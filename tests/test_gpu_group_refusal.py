"""GPU: a group step refused for one member's arguments enqueues nothing on any member.

``lo_group_project_cast_hist_dev``, ``lo_group_hist_u8_cols_dev`` and ``lo_group_minmax_cast_dev`` check every local
member's input before anything is launched.  A call whose last member's input is NULL, of the wrong dtype or short of a
column returns LO_ERR_INVALID with that member's message and launches nothing.  The previous step's result stays
readable, and the next step equals the oracle with no merge timeouts.

A local group of one runs on any GPU machine.  A local group of two needs two visible GPUs and is skipped otherwise.
It is the case that goes wrong when member 0 launches before member 1 is refused: its kernel arrives at a step the
group never finishes.  The root then waits out the merge timeout, and the arrival counter runs one ahead of the
group's own step count.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from edge_values import ref_minmax
from oracle import bsem_numpy as bn

pytestmark = pytest.mark.gpu
ROWS = 20011
NBINS = 64
LO, HI = -1000.0, 1000.0
ENTRIES = {          # entry -> (table dtype, k): u8-65 takes k_group_merge_big, or in a group of one its own shortcut
    "project": ("f64", 3),
    "u8": ("u8", 4),
    "u8-65": ("u8", 65),
    "minmax": ("f64", 3),
}
BAD = ["null", "dtype", "cols"]


@pytest.fixture(scope="module", params=[1, 2], ids=["one-member", "two-members"])
def group(request, built):
    if torch.cuda.device_count() < request.param:
        pytest.skip("a local group of two needs two visible GPUs")
    from learningorchestra_b200.sharding import ShardedEngine
    sh = ShardedEngine.local(list(range(request.param)))
    yield sh
    sh.close()


def _data(name):
    dtype, k = ENTRIES[name]
    rng = np.random.default_rng(k)
    if dtype == "u8":
        return rng.integers(0, 256, (k, ROWS), dtype=np.uint8)
    x = rng.uniform(-1200.0, 1200.0, (k, ROWS))
    x[:, ::101] = np.nan
    x[1, ::37] = np.inf
    return x


def _expected(name, x, col_idx):
    if name == "project":
        return bn.project_cast_hist(x, col_idx, NBINS, np.full(len(col_idx), LO, np.float32),
                                    np.full(len(col_idx), HI, np.float32))[1]
    if name == "minmax":
        return np.array([[np.float32(mn).view(np.uint32), np.float32(mx).view(np.uint32), nf]
                         for mn, mx, nf in map(ref_minmax, x[col_idx])], np.uint64)
    return np.stack([np.bincount(x[c], minlength=256) for c in col_idx]).astype(np.uint64)


def _read(sh, name, k):
    """The last step's merged result on member 0, laid out as ``_expected``."""
    from learningorchestra_b200.engine import _minmax_decode
    if name == "minmax":
        mins, maxs, cnt = _minmax_decode(sh._lib, sh.result(3 * k), k)
        return np.stack([mins.view(np.uint32).astype(np.uint64), maxs.view(np.uint32).astype(np.uint64), cnt], 1)
    return sh.result(k * (NBINS if name == "project" else 256)).reshape(k, -1)


def _step(sh, name, t, col_idx):
    if name == "project":
        sh.project_cast_hist(t, col_idx, NBINS, LO, HI, bcast=True)
    elif name == "minmax":
        sh.minmax_cast(t, col_idx)
    else:
        sh.hist_u8_cols(t, col_idx, bcast=True)
    return _read(sh, name, len(col_idx))


def _call(sh, name, handles, col_idx):
    """The raw entry point over the given member tables: (return code, message)."""
    from learningorchestra_b200 import _native as N
    k = len(col_idx)
    tables = (C.c_void_p * sh.nlocal)(*handles)
    idx = (C.c_int32 * k)(*col_idx)
    if name == "project":
        spec, _keep = sh.engines[0]._spec(k, NBINS, LO, HI)
        rc = sh._lib.lo_group_project_cast_hist_dev(sh._g, tables, idx, k, None, C.byref(spec), N.LO_GROUP_BCAST, None)
    elif name == "minmax":
        rc = sh._lib.lo_group_minmax_cast_dev(sh._g, tables, idx, k, None)
    else:
        rc = sh._lib.lo_group_hist_u8_cols_dev(sh._g, tables, idx, k, N.LO_GROUP_BCAST, None)
    return rc, sh._lib.lo_last_error().decode()


def _message(name, bad, member, k):
    from learningorchestra_b200 import _native as N
    if bad == "cols":
        return f"col_idx[0] = {k - 1} outside [0, {k - 1})"
    if name == "minmax":
        return f"in[{member}] must be an LO_F64 table"
    if bad == "null":
        return f"in[{member}] is NULL"
    if ENTRIES[name][0] == "u8":
        return f"input table must be LO_U8 (got dtype {N.LO_F64})"
    return f"input table must be LO_F64 (got dtype {N.LO_U8})"


@pytest.mark.parametrize("bad", BAD)
@pytest.mark.parametrize("name", list(ENTRIES))
def test_a_refused_member_launches_nothing_and_the_next_step_is_exact(group, name, bad):
    from learningorchestra_b200 import _native as N
    sh = group
    dtype, k = ENTRIES[name]
    col_idx = list(range(k))[::-1]
    x = _data(name)
    want = _expected(name, x, col_idx)
    t = sh.table_from_numpy(x)
    last = sh.nlocal - 1
    rows = t.shards[last].nrows
    other = "u8" if dtype == "f64" else "f64"
    wrong = None if bad == "null" else sh.engines[last].table(other if bad == "dtype" else dtype, rows,
                                                                k if bad == "dtype" else k - 1)
    try:
        np.testing.assert_array_equal(_step(sh, name, t, col_idx), want)
        l0 = sh.launch_count
        rc, msg = _call(sh, name, [s._h for s in t.shards[:last]] + [wrong._h if wrong else None], col_idx)
        assert (rc, msg) == (N.LO_ERR_INVALID, _message(name, bad, last, k))
        assert sh.launch_count == l0
        np.testing.assert_array_equal(_read(sh, name, k), want)       # the refused call left the last result alone
        np.testing.assert_array_equal(_step(sh, name, t, col_idx), want)
        assert sh.timeouts() == 0
    finally:
        if wrong is not None:
            wrong.free()
        t.free()
