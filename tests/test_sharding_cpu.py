"""CPU: the N > 1 host logic — shard bounds and the single count all-reduce — over gloo, world size 2 and 3.
Each rank computes its shard's partial histogram with the ORACLE (there is no GPU here); what is under
test is the sharding arithmetic and the reduction plumbing that bench.py / the executors use on NCCL."""
import os
import socket
import threading
import time

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from learningorchestra_b200.sharding import all_shard_bounds, allreduce_counts, column_batches, on_each, shard_bounds

SEED = 20260921
GROUP_CAP = 262144          # LO_GROUP_MAX_COUNTS


def test_column_batches_fit_the_group_cap():
    from learningorchestra_b200 import _native as N
    assert N.LO_GROUP_MAX_COUNTS == GROUP_CAP
    # within the cap: one step, today's single asynchronous call
    assert column_batches(4, 65536) == [(0, 4)]
    assert column_batches(1024, 256) == [(0, 1024)]
    assert column_batches(64, 4096) == [(0, 64)]
    # over it: runs of cap // nbins columns in column order, the last one short
    assert column_batches(5, 65536) == [(0, 4), (4, 5)]
    assert column_batches(128, 4096) == [(0, 64), (64, 128)]
    assert column_batches(65, 4096) == [(0, 64), (64, 65)]
    assert column_batches(3, 200_000, cap=150_000) == [(0, 1), (1, 2), (2, 3)]     # wider than the cap: one column each
    for k in (1, 2, 5, 17, 64, 65, 127, 128):
        for nbins in (1, 7, 256, 1000, 2048, 2049, 4096, 16384, 16385, 52429, 57345, 65536):
            b = column_batches(k, nbins)
            assert b[0][0] == 0 and b[-1][1] == k
            assert all(e0 == b1 for (_, e0), (b1, _) in zip(b[:-1], b[1:]))          # contiguous, in order
            assert all((e - s) * nbins <= GROUP_CAP for s, e in b)
            assert len(b) == (1 if k * nbins <= GROUP_CAP else -(-k // (GROUP_CAP // nbins)))
            assert b == column_batches(k, nbins)                                     # the same on every rank


def test_shard_bounds_cover_and_align():
    for total in (0, 1, 31, 32, 33, 1000, 100_000_000, 12_345_677):
        for world in (1, 2, 3, 4, 8):
            b = all_shard_bounds(total, world)
            assert b[0][0] == 0 and b[-1][1] == total
            for (a0, a1), (b0, b1) in zip(b[:-1], b[1:]):
                assert a1 == b0 and a0 <= a1
            for (x0, _x1) in b[1:]:
                assert x0 % 32 == 0
    assert shard_bounds(100_000_000, 8, 3) == (37_500_000, 50_000_000)
    with pytest.raises(ValueError):
        shard_bounds(10, 2, 2)


def test_on_each_runs_every_member_at_once_and_undoes_the_results_of_a_failed_fan_out():
    n = 5
    together = threading.Barrier(n, timeout=30)      # breaks unless all members are running at the same time

    def square(i):
        together.wait()
        time.sleep(0.01 * (n - i))                   # the last member finishes first
        return i * i

    assert on_each(n, square) == [i * i for i in range(n)]
    assert on_each(0, square) == []

    ran, undone, lock = [], [], threading.Lock()

    def some_fail(i):
        time.sleep(0.01 * (n - i))
        with lock:
            ran.append(i)
        if i in (1, 3):                              # member 3 raises first, member 1 comes first in member order
            raise ValueError(f"member {i}")
        return {"member": i}

    with pytest.raises(ValueError, match="member 1"):
        on_each(n, some_fail, undo=undone.append)
    assert sorted(ran) == list(range(n))
    assert sorted(r["member"] for r in undone) == [0, 2, 4]
    with pytest.raises(ValueError, match="member 1"):
        on_each(n, some_fail)                        # no undo: the first failure still comes back


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, total_rows, ncols, nbins, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import cport
    r0, r1 = shard_bounds(total_rows, world, rank)
    lo = np.full(ncols, -1000.0, np.float32)
    hi = np.full(ncols, 1000.0, np.float32)
    part, _ = cport.synth_project_cast_hist(1, SEED, r0, r1 - r0, -1000.0, 1000.0, list(range(ncols)), nbins, lo, hi)
    t = torch.from_numpy(part.view(np.int64).copy())
    allreduce_counts(t)
    if rank == 0:
        ret.put(t.numpy().view(np.uint64).copy())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_counts_allreduce_over_gloo(built, world):
    from oracle import cport
    total_rows, ncols, nbins = 250_007, 4, 256
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, total_rows, ncols, nbins, ret)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = ret.get(timeout=240)                       # never block forever if a worker died
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    lo = np.full(ncols, -1000.0, np.float32)
    hi = np.full(ncols, 1000.0, np.float32)
    exp, _ = cport.synth_project_cast_hist(1, SEED, 0, total_rows, -1000.0, 1000.0, list(range(ncols)), nbins, lo, hi)
    np.testing.assert_array_equal(got, exp)
