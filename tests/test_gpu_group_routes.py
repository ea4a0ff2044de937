"""GPU: every route of the multi-GPU group step (``lo_group_*`` / ``ShardedEngine``) against the oracle, at the bin edges.

A group step runs the single-device kernels plus a merge: per-column tickets, system-scope REDs into the root's merge
matrix, and the root's epilogue inside the streaming kernel (k * nbins <= 16 384 counts) or in a second launch,
``k_group_merge_big``.  ``k_group_push`` finishes empty shards, the host pipelines and the min/max pre-pass.  Steps
alternate between two accumulate and merge matrices (parities), and ``independent=True`` lets them overlap.

One spawn per configuration (peer merge at world 1, 2 and 3 on shared devices; NCCL at world 1, and at world 2 when two
GPUs are visible) runs the whole case list on every rank, each route case twice in a row so both parities are used.
The parent compares every step with the oracle: counts exactly, fp32 outputs bit for bit with the oracle's cast, fp64
copies bit for bit with the input.  Every rank also reports the route it took: its launch count (1 for a step whose
epilogue runs in the streaming kernel, 2 with ``k_group_merge_big``, 1 for an empty shard), the tile kernel's IEEE
divide launches, the wide-bin kernel's ``selftest_fastdiv`` flag, and no merge timeouts.

Each column holds the edge values of its own (lo, hi, nbins) (``edge_values.edge_column``); columns of one step have
different ranges, safe and IEEE widths mixed on the IEEE routes.  Row counts put the shard cuts (multiples of 32)
inside tiles and wide-bin rounds.
"""
import ctypes as C
import datetime
import os
import socket
from typing import NamedTuple

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from edge_values import F32_MAX, F32_MAX_TIE, NAN_BITS, edge_column, f64, ref_minmax
from learningorchestra_b200.sharding import all_shard_bounds, column_batches
from oracle import bsem_numpy as bn

CAP = 262144                 # LO_GROUP_MAX_COUNTS: counts every group matrix holds
EPILOGUE_MAX = 16384         # largest matrix whose root epilogue runs inside the streaming kernel
TILE_BINS = 256              # the tile kernel up to here, the wide-bin kernel above
WIDE_SMEM_MAX = 57344        # wide-bin counters in shared memory up to here, in L2 above
TILE = 61440                 # rows per tile of the tile kernel (and per chunk of the host pipeline at 1 MiB)
ROUND = 8192                 # rows per loop round of the wide-bin kernel
W = float(np.uint32(0x3FFFFFFF).view(np.float32))     # 1.9999999: all-ones significand, never the fast divide

R_FEW = 2 * TILE + 4099      # k <= 4: three tiles per column; cuts at 63 488 (world 2), 42 304 / 84 640 (world 3)
R_MANY = 20011               # many columns: cuts at 9 984 (world 2), 6 656 / 13 312 (world 3)
R_EMPTY = 40                 # world 3: cuts at 0, 0 -> the root and rank 1 hold no rows
R_HOST = 3 * (2 * TILE + 1234) + 17   # every rank's shard takes several 1 MiB chunks of two columns
R_MINMAX = 30011

SAFE = [(-1000.0, 1000.0), (-123.456, 789.012), (1e6, 1e6 + 64.0)]
TILE_IEEE = [(0.0, 2.0 ** -93), (-1e38, 1e38)]        # at 256 bins: w = 2^-101, w > 2^100
WIDE_IEEE = [(0.0, 1e-28), (-1e38, 1e38)]             # above 256 bins: w < 2^-100, w > 2^100


class Case(NamedTuple):
    name: str
    kind: str                    # "f64" (device step), "u8", "host" (host pipeline), "batched" (ShardedEngine split)
    kernel: str                  # "tile" | "bins" | "u8"
    divide: str | None           # "edges" | "ieee" | "fast" | None (u8)
    nbins: int
    ranges: tuple                # (lo, hi) of each table column; k = len(ranges)
    rows: int
    out: str | None = None       # None | "f32" | "f64"
    wrapped: bool = False        # input at base + 8 bytes, output at + 4 (f32) / + 8 (f64): the scalar kernels
    bcast: bool = True

    @property
    def k(self):
        return len(self.ranges)

    @property
    def n(self):
        return self.k * self.nbins

    @property
    def epilogue(self):
        return "kernel" if self.n <= EPILOGUE_MAX else "big"

    @property
    def counters(self):
        return None if self.kernel != "bins" else ("smem" if self.nbins <= WIDE_SMEM_MAX else "l2")

    @property
    def col_idx(self):           # projected columns: the table's, reversed
        return list(range(self.k))[::-1]

    @property
    def lo(self):
        return np.array([self.ranges[c][0] for c in self.col_idx], np.float32)

    @property
    def hi(self):
        return np.array([self.ranges[c][1] for c in self.col_idx], np.float32)


def _cols(base, k):
    return tuple(base[j % len(base)] for j in range(k))


def _route_cases():
    """Every (kernel, divide, OUT, aligned, epilogue) once; the wide-bin big matrices alternate their counters."""
    cases = []
    shapes = {   # (kernel, divide, epilogue) -> (nbins, k, column ranges, rows)
        ("tile", "edges", "kernel"): (256, 3, SAFE, R_FEW),
        ("tile", "ieee", "kernel"): (256, 3, TILE_IEEE + SAFE[:1], R_FEW),
        ("tile", "edges", "big"): (256, 65, SAFE, R_MANY),
        ("tile", "ieee", "big"): (256, 65, TILE_IEEE + SAFE, R_MANY),
        ("bins", "fast", "kernel"): (1000, 3, SAFE, R_FEW),
        ("bins", "ieee", "kernel"): (1000, 3, WIDE_IEEE[:1] + SAFE[:2], R_FEW),
    }
    big_wide = {("fast", "smem"): (16384, 2, SAFE[:2]), ("ieee", "smem"): (16384, 2, WIDE_IEEE[:1] + SAFE[:1]),
                ("fast", "l2"): (65536, 2, SAFE[:1] + SAFE[2:]), ("ieee", "l2"): (65536, 3, WIDE_IEEE + SAFE[:1])}
    i = 0
    for kernel, divide in [("tile", "edges"), ("tile", "ieee"), ("bins", "fast"), ("bins", "ieee")]:
        for epilogue in ("kernel", "big"):
            for o, out in enumerate((None, "f32", "f64")):
                for wrapped in (False, True):
                    if (kernel, epilogue) == ("bins", "big"):
                        counters = ("smem", "l2")[(o + wrapped) % 2]
                        nbins, k, base = big_wide[(divide, counters)]
                        rows = R_FEW
                    else:
                        nbins, k, base, rows = shapes[(kernel, divide, epilogue)]
                    layout = "wrap" if wrapped else "aligned"
                    name = f"{kernel}-{divide}-{epilogue}-{out or 'hist'}-{layout}-{k}x{nbins}"
                    cases.append(Case(name, "f64", kernel, divide, nbins, _cols(base, k), rows, out, wrapped,
                                      bcast=i % 2 == 0))
                    i += 1
    return cases


ROUTE_CASES = _route_cases()
BOUNDARY_CASES = [
    Case("tile-edges-64x256", "f64", "tile", "edges", 256, _cols(SAFE, 64), R_MANY, "f32"),
    Case("tile-ieee-64x256", "f64", "tile", "ieee", 256, _cols(TILE_IEEE + SAFE, 64), R_MANY, None, True, False),
    Case("bins-fast-16x1024", "f64", "bins", "fast", 1024, _cols(SAFE, 16), R_MANY, "f32", True),
    Case("bins-ieee-16x1024", "f64", "bins", "ieee", 1024, _cols(WIDE_IEEE + SAFE, 16), R_MANY, "f64"),
    Case("bins-fast-1x16385", "f64", "bins", "fast", 16385, SAFE[:1], R_FEW, "f32"),
    Case("bins-ieee-1x16385", "f64", "bins", "ieee", 16385, WIDE_IEEE[:1], R_FEW, None, False, False),
    Case("bins-fast-4x65536", "f64", "bins", "fast", 65536, _cols(SAFE, 4), R_MANY, "f32", True),
    Case("u8-64", "u8", "u8", None, 256, ((0, 0),) * 64, R_MANY),
    Case("u8-65", "u8", "u8", None, 256, ((0, 0),) * 65, R_MANY, bcast=False),
    Case("u8-1024", "u8", "u8", None, 256, ((0, 0),) * 1024, R_MANY),
]
EMPTY_CASES = [
    Case("empty-tile-edges-2x16", "f64", "tile", "edges", 16, SAFE[:2], R_EMPTY, "f32"),
    Case("empty-tile-ieee-65x256", "f64", "tile", "ieee", 256, _cols(TILE_IEEE + SAFE, 65), R_EMPTY, "f32"),
    Case("empty-bins-fast-1x16385", "f64", "bins", "fast", 16385, SAFE[:1], R_EMPTY, None, False, False),
]
HOST_CASES = [
    Case("host-tile-ieee-2x256", "host", "tile", "ieee", 256, TILE_IEEE[:1] + SAFE[:1], R_HOST, "f32", bcast=False),
    Case("host-bins-ieee-2x65536", "host", "bins", "ieee", 65536, SAFE[:1] + WIDE_IEEE[:1], R_HOST, "f32", bcast=False),
]
BATCHED_CASES = [     # over LO_GROUP_MAX_COUNTS: ShardedEngine splits them into column batches
    Case("batched-5x65536", "batched", "bins", None, 65536, _cols(SAFE + WIDE_IEEE, 5), R_MANY, "f32", bcast=False),
    Case("batched-128x4096", "batched", "bins", None, 4096, _cols(SAFE, 128), R_MANY, "f64", True),
    Case("batched-host-5x65536", "host", "bins", None, 65536, _cols(SAFE + WIDE_IEEE, 5), R_MANY, "f32", bcast=True),
]
CASES = {c.name: c for c in ROUTE_CASES + BOUNDARY_CASES + EMPTY_CASES + HOST_CASES + BATCHED_CASES}
# in-kernel f64, merge_big f64, u8, host pipeline, min/max and an empty-shard step: consecutive steps of one parity take
# different routes, so a matrix one route leaves non-zero shows up in the next step of that parity
MIXED = ["tile-edges-kernel-f64-aligned-3x256", "bins-fast-big-f64-aligned-2x16384", "u8-65", "host-tile-ieee-2x256",
         "minmax", "empty-tile-edges-2x16"]
NCCL_SUBSET = [c.name for c in ROUTE_CASES[::3]] + ["u8-1024", "bins-fast-4x65536"] + [c.name for c in HOST_CASES]
MINMAX_COLUMNS = 7


# ---- the host's route rules, restated (loexec.cu: fastdiv_ok, edges_ok) ------------------------------------------
def _width(lo, hi, nbins):
    return float(bn.bin_width(lo, hi, nbins))


def _edges_ok(w):
    return 2.0 ** -100 <= w <= 2.0 ** 100


def _fastdiv_ok(w):
    return _edges_ok(w) and (int(np.float32(w).view(np.uint32)) & 0x7FFFFF) != 0x7FFFFF


def _divide_of(kernel, ranges, nbins):
    ok = _edges_ok if kernel == "tile" else _fastdiv_ok
    fast = all(ok(_width(lo, hi, nbins)) for lo, hi in ranges)
    return ("edges" if kernel == "tile" else "fast") if fast else "ieee"


# ---- data: every process rebuilds the same columns ---------------------------------------------------------------
_data = {}


def _f64_table(c):
    """[k, rows]: column j holds the edge column of its own range at c.nbins, repeated and rotated by j."""
    if c.name not in _data:
        cols = []
        for j, (lo, hi) in enumerate(c.ranges):
            x = edge_column(lo, hi, c.nbins)
            cols.append(x[(np.arange(c.rows) + 7919 * j) % x.size])
        _data[c.name] = np.stack(cols)
    return _data[c.name]


def _u8_table(c):
    if c.name not in _data:
        x = np.random.default_rng(c.k).integers(0, 256, (c.k, c.rows), dtype=np.uint8)
        x[:, ::97] = 255
        x[:, 1::89] = 0
        _data[c.name] = x
    return _data[c.name]


def _minmax_table(world):
    """Pre-pass columns placed per shard: the first shard only NaN; the last only +-inf; -0.0 on the first shard and +0.0
    on the last; the only finite value in the last row; FLT_MAX ties over every shard; no finite value anywhere."""
    rows = R_MINMAX
    bounds = all_shard_bounds(rows, world)
    (f0, f1), (l0, l1), mid = bounds[0], bounds[-1], bounds[len(bounds) // 2]
    rng = np.random.default_rng(13)
    normal = rng.normal(0.0, 1e4, rows)
    nan = f64(np.array(NAN_BITS, np.uint64)[rng.integers(0, len(NAN_BITS), rows)])
    infs = np.where(rng.random(rows) < 0.5, np.inf, -np.inf)
    ties = np.where(rng.random(rows) < 0.5, F32_MAX_TIE, -F32_MAX_TIE)        # cast to +-inf
    cols = []
    c = normal.copy()
    c[f0:f1] = nan[f0:f1]
    cols.append(c)
    c = normal.copy()
    c[l0:l1] = infs[l0:l1]
    cols.append(c)
    c = nan.copy()
    c[f0] = -0.0
    c[l1 - 1] = 0.0
    cols.append(c)
    c = nan.copy()
    c[l1 - 1] = -12.375
    cols.append(c)
    c = ties.copy()
    c[f0] = F32_MAX
    c[mid[0]] = float(np.nextafter(F32_MAX_TIE, 0.0))                          # casts to FLT_MAX
    c[l1 - 1] = -F32_MAX
    cols.append(c)
    cols.append(np.where(rng.random(rows) < 0.3, nan, np.where(rng.random(rows) < 0.5, infs, ties)))
    cols.append(normal)
    assert len(cols) == MINMAX_COLUMNS
    return np.stack(cols)


# ---- one rank ---------------------------------------------------------------------------------------------------
def _shard_input(sh, eng, local, total, offset, dtype, wrapped):
    """ShardedTable over this rank's rows: aligned, or wrapped at base + 8 bytes with a pitch of rows + 1 elements."""
    from learningorchestra_b200.sharding import ShardedTable
    k, n = local.shape
    if not wrapped:
        t = sh.table(dtype, total, k)
        if n:
            for j in range(k):
                t.upload(j, local[j])
        return t, [t]
    flat = np.zeros(1 + k * (n + 1), local.dtype)
    for j in range(k):
        flat[1 + j * (n + 1): 1 + j * (n + 1) + n] = local[j]
    big = eng.table_from_numpy(flat[None, :])
    view = eng.wrap(dtype, n, k, big.base_ptr + local.itemsize, (n + 1) * local.itemsize)
    return ShardedTable(sh, [view], [offset], total), [view, big]


def _shard_output(sh, eng, out, k, n, total, offset, wrapped):
    from learningorchestra_b200.sharding import ShardedTable
    if out is None:
        return None, []
    if not wrapped:
        t = sh.table(out, total, k)
        return t, [t]
    size = 4 if out == "f32" else 8
    big = eng.table(out, 1 + k * (n + 1), 1)
    view = eng.wrap(out, n, k, big.base_ptr + size, (n + 1) * size)
    return ShardedTable(sh, [view], [offset], total), [view, big]


def _out_mismatches(c, out, local):
    """Elements of this rank's output whose bits differ from the oracle's cast (f32) or from the input (f64)."""
    bad = 0
    for j, col in enumerate(c.col_idx):
        got = out.to_numpy(j)
        want = bn.cast_f64_f32(local[col]) if c.out == "f32" else local[col]
        bad += int((got.view({4: np.uint32, 8: np.uint64}[got.itemsize]) !=
                    want.view({4: np.uint32, 8: np.uint64}[want.itemsize])).sum())
    return bad


def _refused(sh, n):
    """lo_group_result on a rank that received no result: LO_ERR_INVALID."""
    from learningorchestra_b200 import _native as N
    try:
        sh.result(n)
    except N.LoexecError as e:
        return e.code == N.LO_ERR_INVALID
    return False


_fastdiv_flags = {}


def _fastdiv(eng, c):
    out = []
    for lo, hi in sorted(set(c.ranges)):
        key = (lo, hi, c.nbins)
        if key not in _fastdiv_flags:
            _fastdiv_flags[key] = eng.selftest_fastdiv(lo, hi, c.nbins)
        out.append(_fastdiv_flags[key])
    return out


def _device_step(sh, eng, c, rank, runs=2, independent=False):
    x = _f64_table(c) if c.kind != "u8" else _u8_table(c)
    (b, e), = sh.bounds(c.rows)
    local = x[:, b:e]
    t, free = _shard_input(sh, eng, local, c.rows, b, "u8" if c.kind == "u8" else "f64", c.wrapped)
    out, free_out = _shard_output(sh, eng, c.out, c.k, e - b, c.rows, b, c.wrapped)
    res = []
    for _ in range(runs):
        l0, d0 = eng.launch_count, eng.edge_tables_info()[2]
        if c.kind == "u8":
            counts = sh.hist_u8_cols(t, c.col_idx, bcast=c.bcast, independent=independent)
        else:
            counts = sh.project_cast_hist(t, c.col_idx, c.nbins, c.lo, c.hi, out=out, bcast=c.bcast,
                                          independent=independent)
        r = {"rows": e - b, "launches": eng.launch_count - l0, "divide": eng.edge_tables_info()[2] - d0}
        holds = c.bcast or rank == 0 or sh.merge == "nccl"
        r["counts"] = counts.to_numpy() if holds else None
        if not holds:
            r["refused"] = _refused(sh, min(c.n, CAP))
            if c.kind == "batched":
                try:
                    counts.to_numpy()
                    r["batched_refused"] = False
                except Exception:
                    r["batched_refused"] = True
        if out is not None:
            r["out_bad"] = _out_mismatches(c, out, local)
        r["timeouts"] = sh.timeouts()
        res.append(r)
    if c.kernel == "bins" and c.kind == "f64":
        res[0]["fastdiv"] = _fastdiv(eng, c)
    for d in free_out + free:
        d.free()
    return res


def _host_step(sh, eng, c, rank):
    x = _f64_table(c)
    (b, e), = sh.bounds(c.rows)
    cols = [np.ascontiguousarray(x[col, b:e]) for col in c.col_idx]
    outs = [np.empty(e - b, np.float32) for _ in cols]
    l0, d0 = eng.launch_count, eng.edge_tables_info()[2]
    counts, tm = sh.project_cast_hist_host(cols, c.nbins, c.lo, c.hi, out=outs, bcast=c.bcast)
    r = {"rows": e - b, "launches": eng.launch_count - l0, "divide": eng.edge_tables_info()[2] - d0,
         "chunks": tm["launches"], "counts": counts if (c.bcast or rank == 0 or sh.merge == "nccl") else None,
         "out_bad": sum(int((o.view(np.uint32) != bn.cast_f64_f32(v).view(np.uint32)).sum()) for o, v in zip(outs, cols)),
         "timeouts": sh.timeouts()}
    if c.kernel == "bins" and c.divide:
        r["fastdiv"] = _fastdiv(eng, c)
    return [r]


def _minmax_step(sh, eng, world, runs=2):
    x = _minmax_table(world)
    (b, e), = sh.bounds(R_MINMAX)
    t, free = _shard_input(sh, eng, x[:, b:e], R_MINMAX, b, "f64", False)
    res = []
    for _ in range(runs):
        mins, maxs, cnt = sh.minmax_cast(t, range(MINMAX_COLUMNS))
        res.append({"mins": mins.view(np.uint32).tolist(), "maxs": maxs.view(np.uint32).tolist(),
                    "cnt": [int(v) for v in cnt], "timeouts": sh.timeouts()})
    for d in free:
        d.free()
    return res


def _contracts(sh, eng):
    """k * nbins = LO_GROUP_MAX_COUNTS + 1 at the ABI, device and host entry points: refused, nothing launched."""
    from learningorchestra_b200 import _native as N
    lib = N.load()
    k, nbins = 5, 52429
    assert k * nbins == CAP + 1
    t = sh.table("f64", 64, k)
    spec, _keep = eng._spec(k, nbins, -1000.0, 1000.0)
    idx = (C.c_int32 * k)(*range(k))
    host_cols = [np.zeros(10) for _ in range(k)]
    in_p = (C.c_void_p * k)(*[a.ctypes.data for a in host_cols])
    counts = np.zeros(k * nbins, np.uint64)
    l0 = eng.launch_count
    rc_dev = lib.lo_group_project_cast_hist_dev(sh._g, sh._tables(t), idx, k, None, C.byref(spec), N.LO_GROUP_BCAST, None)
    msg_dev = lib.lo_last_error().decode()
    rc_host = lib.lo_group_project_cast_hist_host(sh._g, in_p, 10, k, None, C.byref(spec),
                                                  counts.ctypes.data_as(C.c_void_p), 0, None)
    msg_host = lib.lo_last_error().decode()
    got = {"rc": [rc_dev, rc_host], "msg": [msg_dev, msg_host], "launches": eng.launch_count - l0}
    t.free()
    return got


def _worker(rank, world, port, merge, names, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["LOEXEC_CHUNK_MB"] = "1"          # the host pipelines take several chunks per shard
    dev = rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    from learningorchestra_b200.engine import Engine
    from learningorchestra_b200.sharding import ShardedEngine
    got = {}
    eng = Engine(dev)
    sh = ShardedEngine.from_torch_distributed(eng, merge=merge)
    try:
        got["merge"] = sh.merge
        dist.barrier()
        got["contracts"] = _contracts(sh, eng)
        for name in names:
            dist.barrier()
            c = CASES[name]
            got[name] = _host_step(sh, eng, c, rank) if c.kind == "host" else _device_step(sh, eng, c, rank)
        dist.barrier()
        got["minmax"] = _minmax_step(sh, eng, world)
        if merge == "peer":
            for independent in (False, True):
                seq = []
                for name in MIXED:
                    dist.barrier()
                    if name == "minmax":
                        seq.append(_minmax_step(sh, eng, world, runs=1)[0])
                    elif CASES[name].kind == "host":
                        seq.append(_host_step(sh, eng, CASES[name], rank)[0])
                    else:
                        seq.append(_device_step(sh, eng, CASES[name], rank, runs=1, independent=independent)[0])
                got[f"mixed-{independent}"] = seq
        dist.barrier()
    except Exception:
        import traceback
        got["error"] = traceback.format_exc()
    ret.put((rank, got))
    try:
        dist.barrier()
    finally:
        sh.close()
        eng.close()
        dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


_runs = {}


def _run(world, merge):
    """Every rank's report of the whole case list, spawned once per configuration."""
    key = (world, merge)
    if key not in _runs:
        names = list(CASES) if merge == "peer" else NCCL_SUBSET
        ctx = mp.get_context("spawn")
        ret = ctx.Queue()
        port = _free_port()
        procs = [ctx.Process(target=_worker, args=(r, world, port, merge, names, ret)) for r in range(world)]
        for p in procs:
            p.start()
        res = {}
        try:
            for _ in range(world):
                r, got = ret.get(timeout=600)        # never block forever if a worker died
                res[r] = got
        finally:
            for p in procs:
                p.join(timeout=60)
                if p.is_alive():
                    p.kill()
        for r in sorted(res):
            assert "error" not in res[r], f"rank {r}:\n{res[r]['error']}"
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
        _runs[key] = (names, res)
    return _runs[key]


# ---- the parent's checks ----------------------------------------------------------------------------------------
_oracle = {}


def _expected(c):
    if c.name not in _oracle:
        if c.kind == "u8":
            x = _u8_table(c)
            _oracle[c.name] = np.stack([np.bincount(x[col], minlength=256) for col in c.col_idx]).astype(np.uint64)
        else:
            _oracle[c.name] = bn.project_cast_hist(_f64_table(c), c.col_idx, c.nbins, c.lo, c.hi)[1]
    return _oracle[c.name]


def _flag_waits(c, rank, merge):
    """lo_group_result's wait for the root's epilogue: one launch per step a peer reads within the call itself (the
    column batches of a split request)."""
    return len(column_batches(c.k, c.nbins)) if merge == "peer" and rank > 0 and c.bcast else 0


def _expected_launches(c, rows, world, merge, rank):
    if c.kind == "batched":
        steps = len(column_batches(c.k, c.nbins))
        per = 1 if merge == "nccl" else 2
        return (steps * per if rows else (0 if merge == "nccl" else steps)) + _flag_waits(c, rank, merge)
    if merge == "nccl":
        return 1 if rows else 0
    if not rows:
        return 1
    if c.kind == "u8" and world == 1 and c.epilogue == "big":
        return 1                                    # a group of one counts straight into its result
    return 2 if c.epilogue == "big" else 1


def _check_step(c, r, rank, world, merge, fails, where):
    def bad(msg):
        fails.append(f"{where} rank {rank}: {msg}")
    if r["counts"] is not None and not np.array_equal(r["counts"], _expected(c)):
        diff = np.argwhere(r["counts"] != _expected(c))
        bad(f"counts differ from the oracle at {len(diff)} entries, first [col, bin] {diff[0].tolist()}")
    if r["counts"] is None and (c.bcast or rank == 0 or merge == "nccl"):
        bad("no counts")
    if "refused" in r and not (r["refused"] and r.get("batched_refused", True)):
        bad("a rank without the result read one after a root-only step")
    if r.get("out_bad"):
        bad(f"{r['out_bad']} output elements differ from the oracle")
    if r["timeouts"]:
        bad(f"{r['timeouts']} merge timeouts")
    if c.kind == "host":
        if r["chunks"] < (2 if c.rows == R_HOST else 1):
            bad(f"{r['chunks']} chunks")
        extra = 0 if merge == "nccl" else len(column_batches(c.k, c.nbins))     # one push / merge_big per step
        if r["launches"] != r["chunks"] + extra + _flag_waits(c, rank, merge):
            bad(f"{r['launches']} launches for {r['chunks']} chunks")
        if c.divide and r["divide"] != (r["chunks"] if (c.kernel, c.divide) == ("tile", "ieee") else 0):
            bad(f"{r['divide']} IEEE-divide tile launches")
    else:
        want = _expected_launches(c, r["rows"], world, merge, rank)
        if r["launches"] != want:
            bad(f"{r['launches']} launches, the {c.epilogue} route takes {want}")
        if c.kind == "f64":
            want_div = 1 if (c.kernel, c.divide) == ("tile", "ieee") and r["rows"] else 0
            if r["divide"] != want_div:
                bad(f"{r['divide']} IEEE-divide tile launches, want {want_div}")
    if "fastdiv" in r:
        flags = r["fastdiv"]
        if not all(b == 0 for used, b in flags if used):
            bad(f"fast divide differs from IEEE: {flags}")
        if all(used for used, _ in flags) != (c.divide == "fast"):
            bad(f"wide-bin divide flags {flags} are not the {c.divide} route")


def _check_minmax(r, world, where, fails):
    x = _minmax_table(world)
    for j in range(MINMAX_COLUMNS):
        mn, mx, nf = ref_minmax(x[j])
        want = (int(np.float32(mn).view(np.uint32)), int(np.float32(mx).view(np.uint32)), nf)
        got = (r["mins"][j], r["maxs"][j], r["cnt"][j])
        if got != want:
            fails.append(f"{where} column {j}: (min, max, finite) bits {got}, oracle {want}")
    if r["timeouts"]:
        fails.append(f"{where}: {r['timeouts']} merge timeouts")


def _check_run(world, merge, select):
    names, res = _run(world, merge)
    fails = []
    for rank, got in res.items():
        assert got["merge"] == merge
        for name in names:
            if select(CASES[name]):
                for i, r in enumerate(got[name]):
                    _check_step(CASES[name], r, rank, world, merge, fails, f"{name} run {i}")
    assert not fails, "\n".join(fails[:40])


CONFIGS = [(1, "peer"), (2, "peer"), (3, "peer")]


@pytest.mark.gpu
@pytest.mark.parametrize("world,merge", CONFIGS, ids=[f"{m}-{w}" for w, m in CONFIGS])
def test_every_route_and_epilogue_boundary_equals_the_oracle(built, world, merge):
    _check_run(world, merge, lambda c: c.kind in ("f64", "u8"))


@pytest.mark.gpu
@pytest.mark.parametrize("world,merge", CONFIGS, ids=[f"{m}-{w}" for w, m in CONFIGS])
def test_host_pipelines_in_a_group_take_several_chunks(built, world, merge):
    _check_run(world, merge, lambda c: c.kind == "host" and c.divide is not None)


@pytest.mark.gpu
@pytest.mark.parametrize("world,merge", CONFIGS, ids=[f"{m}-{w}" for w, m in CONFIGS])
def test_requests_over_the_group_cap_are_split_into_column_batches(built, world, merge):
    _check_run(world, merge, lambda c: c.name.startswith("batched"))


@pytest.mark.gpu
@pytest.mark.parametrize("world,merge", CONFIGS, ids=[f"{m}-{w}" for w, m in CONFIGS])
def test_one_past_the_cap_is_refused_before_any_launch(built, world, merge):
    from learningorchestra_b200 import _native as N
    _, res = _run(world, merge)
    for rank, got in res.items():
        cc = got["contracts"]
        assert cc["rc"] == [N.LO_ERR_INVALID, N.LO_ERR_INVALID], (rank, cc)
        assert cc["launches"] == 0, (rank, cc)
        assert all("262145" in m and "262144" in m for m in cc["msg"]), (rank, cc)
    # the steps after it (the whole case list) still equal the oracle
    _check_run(world, merge, lambda c: c.name == ROUTE_CASES[0].name)


@pytest.mark.gpu
@pytest.mark.parametrize("world,merge", CONFIGS, ids=[f"{m}-{w}" for w, m in CONFIGS])
def test_minmax_over_shards_with_edge_values_split_across_them(built, world, merge):
    _, res = _run(world, merge)
    fails = []
    for rank, got in res.items():
        for i, r in enumerate(got["minmax"]):
            _check_minmax(r, world, f"minmax run {i} rank {rank}", fails)
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("world,merge", CONFIGS, ids=[f"{m}-{w}" for w, m in CONFIGS])
@pytest.mark.parametrize("independent", [False, True])
def test_mixed_sequence_of_routes_on_both_parities(built, world, merge, independent):
    _, res = _run(world, merge)
    fails = []
    for rank, got in res.items():
        for i, (name, r) in enumerate(zip(MIXED, got[f"mixed-{independent}"])):
            if name == "minmax":
                _check_minmax(r, world, f"mixed step {i} (minmax) rank {rank}", fails)
            else:
                _check_step(CASES[name], r, rank, world, merge, fails, f"mixed step {i} ({name})")
    assert not fails, "\n".join(fails[:40])


@pytest.mark.gpu
def test_nccl_merge_on_a_subset_of_routes(built):
    world = 2 if torch.cuda.device_count() >= 2 else 1
    _check_run(world, "nccl", lambda c: True)
    _, res = _run(world, "nccl")
    fails = []
    for rank, got in res.items():
        for i, r in enumerate(got["minmax"]):
            _check_minmax(r, world, f"minmax run {i} rank {rank}", fails)
    assert not fails, "\n".join(fails)


# ---- without a GPU: what the case list reaches -------------------------------------------------------------------
def test_group_case_list_reaches_every_route_and_both_sides_of_every_boundary():
    f64 = [c for c in ROUTE_CASES + BOUNDARY_CASES + EMPTY_CASES if c.kind == "f64"]
    # every (kernel, divide, OUT, aligned, epilogue route), and each one's declared divide is the one the host picks
    seen = {(c.kernel, c.divide, c.out, not c.wrapped, c.epilogue) for c in ROUTE_CASES}
    for kernel, divides in (("tile", ("edges", "ieee")), ("bins", ("fast", "ieee"))):
        for divide in divides:
            for out in (None, "f32", "f64"):
                for aligned in (True, False):
                    for epilogue in ("kernel", "big"):
                        assert (kernel, divide, out, aligned, epilogue) in seen, (kernel, divide, out, aligned, epilogue)
    for c in f64 + HOST_CASES:
        assert (c.nbins <= TILE_BINS) == (c.kernel == "tile"), c.name
        if c.divide:
            assert _divide_of(c.kernel, c.ranges, c.nbins) == c.divide, c.name
        if c.divide == "ieee":        # safe and IEEE widths mixed: one IEEE column takes the whole launch
            assert len({_divide_of(c.kernel, [r], c.nbins) for r in c.ranges}) == 2 or c.k == 1, c.name
        assert c.k == 1 or len(set(c.ranges)) > 1, c.name           # columns of one step have different ranges
    # both wide-bin counter routes, each with both divides; L2 always goes through merge_big
    assert {(c.counters, c.divide) for c in f64 if c.kernel == "bins"} >= {(r, d) for r in ("smem", "l2")
                                                                           for d in ("fast", "ieee")}
    assert all(c.epilogue == "big" for c in f64 if c.counters == "l2")
    # both sides of every epilogue boundary, for the tile kernel, the wide-bin kernel and u8; the cap itself
    shapes = {(c.kernel, c.k, c.nbins) for c in CASES.values()}
    for shape in [("tile", 64, 256), ("tile", 65, 256), ("bins", 16, 1024), ("bins", 1, 16385), ("u8", 64, 256),
                  ("u8", 65, 256), ("u8", 1024, 256), ("bins", 4, 65536)]:
        assert shape in shapes, shape
    assert CASES["tile-edges-64x256"].n == EPILOGUE_MAX == CASES["bins-fast-16x1024"].n == CASES["u8-64"].n
    assert CASES["bins-fast-1x16385"].n == EPILOGUE_MAX + 1 and CASES["u8-65"].epilogue == "big"
    assert CASES["u8-1024"].n == CAP == CASES["bins-fast-4x65536"].n
    # an empty shard on the root and on a peer at world 3, on both epilogue routes
    assert all_shard_bounds(R_EMPTY, 3)[:2] == [(0, 0), (0, 0)]
    assert {c.epilogue for c in EMPTY_CASES} == {"kernel", "big"}
    # shard cuts fall inside tiles and wide-bin rounds, and no shard is empty outside the empty-shard cases
    for c in CASES.values():
        if c.rows == R_EMPTY:
            continue
        for world in (2, 3):
            for b, e in all_shard_bounds(c.rows, world):
                assert e > b and b % 32 == 0 and (b == 0 or (b % ROUND and b % TILE)), (c.name, world, b)
    # results delivered everywhere and to the root only; host pipelines on the IEEE route and through merge_big
    assert {c.bcast for c in f64} == {True, False}
    assert {(c.divide, c.epilogue) for c in HOST_CASES} == {("ieee", "kernel"), ("ieee", "big")}
    assert {c.kernel for c in HOST_CASES} == {"tile", "bins"}
    # the split requests are over the cap; the mixed sequence alternates its routes on each parity
    assert all(c.n > CAP for c in BATCHED_CASES)
    assert len(MIXED) % 2 == 0 and len(MIXED) == len(set(MIXED))
    kinds = [("minmax" if n == "minmax" else "empty" if CASES[n].rows == R_EMPTY else
              CASES[n].kind + "-" + CASES[n].epilogue) for n in MIXED]
    assert set(kinds) == {"f64-kernel", "f64-big", "u8-big", "host-kernel", "minmax", "empty"}
    assert all(n in CASES for n in NCCL_SUBSET)
