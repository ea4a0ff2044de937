"""GPU: every launch route of the binned projection / cast / histogram kernels against the oracle, at and around every
bin edge.

The host picks the kernel from the bin count (the tile kernel up to 256 bins; above, the wide-bin kernel with its counters
in shared memory up to 57 344 bins and in L2 beyond), the divide from each column's bin width (edge table or fast divide
while the width allows it, the IEEE divide otherwise), the instantiation from the output type, and the vector or scalar
path from the slabs' alignment.  Every case names its route and asserts that it got there: the tile kernel through the
context's count of divide launches, the wide-bin kernel through ``selftest_fastdiv``, whose flag is the condition the
launcher tests.  Counts must equal the oracle's, fp32 outputs must be bit-equal to its cast and fp64 copies bit-equal to
the input, NaN payloads included.
"""
from typing import NamedTuple

import numpy as np
import pytest

from edge_values import edge_column
from oracle import bsem_numpy as bn

pytestmark = pytest.mark.gpu

W = float(np.uint32(0x3FFFFFFF).view(np.float32))     # 1.9999999: an all-ones significand (Markstein's exception)
TILE = 61440                                           # rows per tile of the tile kernel
ROUND = 8192                                           # rows per loop round (and here per chunk) of the wide-bin kernel
WIDE_SMEM_MAX = 57344                                  # bins of the largest wide-bin histogram kept in shared memory
MAX_K = 8                                              # columns a case spreads its values over

# (lo, hi, nbins) per (kernel, divide, counters); widths computed as the host does (bn.bin_width)
RANGES = {
    ("tile", "edges", None): [(-1000.0, 1000.0, 256), (-123.456, 789.012, 7), (1e6, 1e6 + 64.0, 256)],
    ("tile", "ieee", None): [(0.0, 2.0 ** -93, 256), (-1e38, 1e38, 7)],                  # w = 2^-101, w > 2^100
    ("bins", "fast", "smem"): [(-1000.0, 1000.0, 512), (-123.456, 789.012, 1000), (1e6, 1e6 + 64.0, 16384),
                               (-1000.0, 1000.0, 40000), (-123.456, 789.012, 57344)],
    ("bins", "fast", "l2"): [(1e6, 1e6 + 64.0, 57345), (-1000.0, 1000.0, 65536)],
    ("bins", "ieee", "smem"): [(0.0, W * 512, 512), (0.0, 1e-28, 1000), (0.0, W * 16384, 16384), (0.0, 1e-28, 40000)],
    ("bins", "ieee", "l2"): [(-1e38, 1e38, 57345), (0.0, W * 65536, 65536)],           # w > 2^100, w = W
}
# the exhaustive fast-divide self-test above 256 bins: w at both ends of the window (2^-100, 2^100), lo far from 0
WIDE_SELFTEST = [(-1000.0, 1000.0, 257), (0.0, 2.0 ** -91, 512), (-(2.0 ** 115), 2.0 ** 115, 65536),
                 (1e6, 1e6 + 64.0, 4096), (1e6, 1e6 + 64.0, 65536), (-123.456, 789.012, 40000), (1e30, 1.5e30, 30000),
                 (-3e7, -2.9e7, 57345)]
# every range the file uses (tests/test_edges_cpu.py pins their edges without a GPU)
EDGE_RANGES = sorted({r for rs in RANGES.values() for r in rs} | set(WIDE_SELFTEST))

# (output, layout): no output takes "in+8" only; "out+4" is an aligned input with an f32 output at +4 bytes
PAIRS = [(None, "aligned"), (None, "in+8"), ("f32", "aligned"), ("f32", "in+8"), ("f32", "out+4"), ("f64", "aligned"),
         ("f64", "in+8")]
# one row; less than one wide-bin round; several wide-bin rounds with a ragged last one; two full tiles, then a tile whose
# first threads take the batch path and the rest the element-wise tail
ROWS = [1, 5003, 5 * ROUND + 17, 2 * TILE + 4099]


class Route(NamedTuple):
    kernel: str
    divide: str
    counters: str | None
    lo: float
    hi: float
    nbins: int
    out: str | None
    layout: str
    rows: int

    @property
    def id(self):
        route = "-".join([self.kernel, self.divide] + ([self.counters] if self.counters else []))
        return f"{route}-{self.out or 'hist'}-{self.layout}-r{self.rows}-({self.lo:.8g},{self.hi:.8g},{self.nbins})"


def _route_matrix():
    """Per (kernel, divide): every (output, layout) pair meets every row shape once.  The wide-bin kernel alternates its
    counter route over both indices, so each route also meets every pair and every row shape."""
    cases, turn = [], {}
    for kernel, divide in [("tile", "edges"), ("tile", "ieee"), ("bins", "fast"), ("bins", "ieee")]:
        for p, (out, layout) in enumerate(PAIRS):
            for r, rows in enumerate(ROWS):
                counters = None if kernel == "tile" else ("smem", "l2")[(p + r) % 2]
                key = (kernel, divide, counters)
                i = turn[key] = turn.get(key, -1) + 1
                cases.append(Route(kernel, divide, counters, *RANGES[key][i % len(RANGES[key])], out, layout, rows))
    return cases


HIST_CASES = _route_matrix()
CAST_CASES = [(out, layout, rows) for out, layout in PAIRS if out for rows in ROWS]


def _bits(a):
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def _table(lo, hi, nbins, rows):
    """[k, rows] fp64: the edge column tiled over k <= MAX_K columns (all of it once there are enough rows)."""
    x = edge_column(lo, hi, nbins)
    k = min(MAX_K, -(-x.size // rows))
    return np.resize(x, k * rows).reshape(k, rows)


def _input(engine, x, layout):
    """(device table of x, tables to free): aligned, or wrapped at base + 8 bytes with a pitch of rows + 1 elements."""
    if layout != "in+8":
        t = engine.table_from_numpy(x)
        return t, [t]
    k, rows = x.shape
    flat = np.zeros(1 + k * (rows + 1))
    for j in range(k):
        flat[1 + j * (rows + 1): 1 + j * (rows + 1) + rows] = x[j]
    big = engine.table_from_numpy(flat[None, :])
    view = engine.wrap("f64", rows, k, big.base_ptr + 8, (rows + 1) * 8)
    return view, [view, big]


def _output(engine, out, k, rows, layout):
    if out is None:
        return None, []
    if layout != "out+4":
        t = engine.table(out, rows, k)
        return t, [t]
    big = engine.table("f32", 1 + k * (rows + 1), 1)
    view = engine.wrap("f32", rows, k, big.base_ptr + 4, (rows + 1) * 4)
    return view, [view, big]


def _check_out(out, x, cast):
    for j in range(x.shape[0]):
        want = x[j] if out.np_dtype == np.float64 else cast[j]
        np.testing.assert_array_equal(_bits(out.to_numpy(j)), _bits(want), err_msg=f"column {j}")


_fastdiv_cache = {}


def _fastdiv(engine, lo, hi, nbins):
    """(the wide-bin launcher takes the fast divide for this range, fp32 patterns where it differs from IEEE)."""
    key = (lo, hi, nbins)
    if key not in _fastdiv_cache:
        _fastdiv_cache[key] = engine.selftest_fastdiv(lo, hi, nbins)
    return _fastdiv_cache[key]


def _divide_launches(engine):
    return engine.edge_tables_info()[2]


def _assert_route(engine, kernel, divide, nbins, ranges, divide_launches):
    """The launch just made reached (kernel, divide); divide_launches: tile launches that took the IEEE divide."""
    if kernel == "tile":
        assert nbins <= 256
        assert divide_launches == (1 if divide == "ieee" else 0)
    else:
        assert nbins > 256 and divide_launches == 0
        flags = [_fastdiv(engine, lo, hi, nbins) for lo, hi in ranges]
        assert all(bad == 0 for used, bad in flags if used)
        assert all(used for used, _ in flags) == (divide == "fast")


def test_route_matrix_reaches_every_instantiation():
    """Every (kernel, OUT, divide, aligned) instantiation of the histogram kernels, and each wide-bin counter route,
    meets every row shape; every wide-bin (OUT, divide, aligned, counters) is reached."""
    def aligned(c):
        return c.layout == "aligned"
    seen = {(c.kernel, c.out, c.divide, aligned(c), c.rows) for c in HIST_CASES}
    for kernel, divide, _ in RANGES:
        for out in (None, "f32", "f64"):
            for al in (True, False):
                assert all((kernel, out, divide, al, rows) in seen for rows in ROWS), (kernel, out, divide, al)
    counters = {(c.counters, c.rows) for c in HIST_CASES if c.kernel == "bins"}
    assert counters == {(route, rows) for route in ("smem", "l2") for rows in ROWS}
    wide = {(c.out, c.divide, aligned(c), c.counters) for c in HIST_CASES if c.kernel == "bins"}
    assert len(wide) == 3 * 2 * 2 * 2
    for c in HIST_CASES:
        assert (c.nbins <= 256) == (c.kernel == "tile")
        assert c.kernel == "tile" or (c.nbins <= WIDE_SMEM_MAX) == (c.counters == "smem")
    assert {(out, layout == "aligned", rows) for out, layout, rows in CAST_CASES} == \
        {(out, al, rows) for out in ("f32", "f64") for al in (True, False) for rows in ROWS}


@pytest.mark.parametrize("case", HIST_CASES, ids=[c.id for c in HIST_CASES])
def test_histogram_route_counts_every_edge_like_the_oracle(engine, case):
    x = _table(case.lo, case.hi, case.nbins, case.rows)
    k = x.shape[0]
    lo = np.full(k, case.lo, np.float32)
    hi = np.full(k, case.hi, np.float32)
    t, free = _input(engine, x, case.layout)
    out, free_out = _output(engine, case.out, k, case.rows, case.layout)
    d0 = _divide_launches(engine)
    counts = engine.project_cast_hist(t, range(k), case.nbins, lo, hi, out=out)
    _assert_route(engine, case.kernel, case.divide, case.nbins, [(case.lo, case.hi)], _divide_launches(engine) - d0)
    cast, want = bn.project_cast_hist(x, range(k), case.nbins, lo, hi)
    np.testing.assert_array_equal(counts.to_numpy(), want)
    if out is not None:
        _check_out(out, x, cast)
    counts.free()
    for d in free_out + free:
        d.free()


@pytest.mark.parametrize("out,layout,rows", CAST_CASES, ids=[f"{o}-{l}-r{r}" for o, l, r in CAST_CASES])
def test_cast_route_without_histogram(engine, out, layout, rows):
    x = _table(0.0, W * 512, 512, rows)
    k = x.shape[0]
    t, free = _input(engine, x, layout)
    o, free_out = _output(engine, out, k, rows, layout)
    d0 = _divide_launches(engine)
    engine.project_cast(t, range(k), out=o)
    assert _divide_launches(engine) == d0
    _check_out(o, x, bn.cast_f64_f32(x))
    for d in free_out + free:
        d.free()


@pytest.mark.parametrize("kernel,nbins,safe,unsafe", [
    ("tile", 256, (-1000.0, 1000.0), (0.0, 2.0 ** -93)),
    ("bins", 1000, (-123.456, 789.012), (0.0, 1e-28)),
    ("bins", 65536, (-1000.0, 1000.0), (0.0, W * 65536)),
])
def test_one_unsafe_width_takes_the_whole_launch_to_the_ieee_divide(engine, kernel, nbins, safe, unsafe):
    rows = 5 * ROUND + 17
    x = np.stack([_table(*safe, nbins, rows)[0], _table(*unsafe, nbins, rows)[0]])
    lo = np.array([safe[0], unsafe[0]], np.float32)
    hi = np.array([safe[1], unsafe[1]], np.float32)
    t = engine.table_from_numpy(x)
    out = engine.table("f32", rows, 2)
    d0 = _divide_launches(engine)
    counts = engine.project_cast_hist(t, [0, 1], nbins, lo, hi, out=out)
    _assert_route(engine, kernel, "ieee", nbins, [safe, unsafe], _divide_launches(engine) - d0)
    if kernel == "bins":
        assert _fastdiv(engine, *safe, nbins)[0]
    cast, want = bn.project_cast_hist(x, [0, 1], nbins, lo, hi)
    np.testing.assert_array_equal(counts.to_numpy(), want)
    _check_out(out, x, cast)
    counts.free(); out.free(); t.free()


def test_columns_past_one_launch_take_their_own_divide(engine):
    """130 columns at 1 000 bins are two launches: 128 columns whose widths take the fast divide, then two that need the
    IEEE divide.  The second launch's counts and outputs start at column 128."""
    nbins, rows = 1000, ROUND + 17
    x = np.stack([_table(-1000.0, 1000.0, nbins, rows)[0], _table(0.0, 1e-28, nbins, rows)[0]])
    cols = [0] * 128 + [1, 1]
    lo = np.array([-1000.0 + j for j in range(128)] + [0.0, 0.0], np.float32)
    hi = np.array([1000.0 + j for j in range(128)] + [1e-28, 2e-28], np.float32)
    assert {float(bn.bin_width(a, b, nbins)) for a, b in zip(lo[:128], hi[:128])} == {2.0}   # one width, shifted ranges
    used, bad = _fastdiv(engine, -1000.0, 1000.0, nbins)
    assert used and bad == 0
    assert not _fastdiv(engine, 0.0, 1e-28, nbins)[0] and not _fastdiv(engine, 0.0, 2e-28, nbins)[0]
    t = engine.table_from_numpy(x)
    out = engine.table("f32", rows, len(cols))
    counts = engine.project_cast_hist(t, cols, nbins, lo, hi, out=out)
    cast, want = bn.project_cast_hist(x, cols, nbins, lo, hi)
    np.testing.assert_array_equal(counts.to_numpy(), want)
    for j in (0, 1, 127, 128, 129):
        np.testing.assert_array_equal(_bits(out.to_numpy(j)), _bits(cast[j]), err_msg=f"column {j}")
    counts.free(); out.free(); t.free()


@pytest.mark.parametrize("lo,hi,nbins", [(0.0, 2.0 ** -93, 256), (-123.456, 789.012, 7), (0.0, W * 512, 512),
                                         (-1000.0, 1000.0, 65536)])
def test_counts_accumulate_over_calls(engine, lo, hi, nbins):
    x = _table(lo, hi, nbins, 5 * ROUND + 17)
    k = x.shape[0]
    t = engine.table_from_numpy(x)
    counts = engine.counts(k, nbins)
    for _ in range(2):
        engine.project_cast_hist(t, range(k), nbins, lo, hi, counts=counts)
    _, want = bn.project_cast_hist(x, range(k), nbins, [lo] * k, [hi] * k)
    np.testing.assert_array_equal(counts.to_numpy(), 2 * want)
    counts.free(); t.free()


@pytest.mark.parametrize("lo,hi,nbins", WIDE_SELFTEST)
def test_fast_divide_is_ieee_divide_exhaustively_at_wide_bins(engine, lo, hi, nbins):
    """All 2^32 fp32 bit patterns: the wide-bin kernel's fast divide bins like __fdiv_rn, the last bin's clamp included."""
    used, bad = engine.selftest_fastdiv(lo, hi, nbins)
    assert used and bad == 0


@pytest.mark.parametrize("lo,hi,nbins", RANGES[("bins", "ieee", "smem")] + RANGES[("bins", "ieee", "l2")])
def test_unsafe_wide_widths_take_the_ieee_divide(engine, lo, hi, nbins):
    assert not engine.selftest_fastdiv(lo, hi, nbins)[0]


@pytest.mark.parametrize("nbins,ranges,fast", [
    (512, [(0.0, W * 512), (-1000.0, 1000.0)], False),            # IEEE divide, shared-memory counters
    (65536, [(-1000.0, 1000.0), (0.0, W * 65536)], False),        # IEEE divide, L2 counters
    (57345, [(1e6, 1e6 + 64.0), (-123.456, 789.012)], True),      # fast divide, L2 counters
])
def test_host_pipeline_chunks_through_the_wide_bin_routes(engine, monkeypatch, nbins, ranges, fast):
    """1 MiB chunks: two columns go through five chunks of 61 440 rows (the last one short), one launch each."""
    monkeypatch.setenv("LOEXEC_CHUNK_MB", "1")
    rows = 4 * TILE + 1234
    x = np.stack([np.resize(edge_column(lo, hi, nbins), rows) for lo, hi in ranges])
    lo = np.array([r[0] for r in ranges], np.float32)
    hi = np.array([r[1] for r in ranges], np.float32)
    outs = [np.empty(rows, np.float32) for _ in ranges]
    counts, timing = engine.project_cast_hist_host([x[0], x[1]], nbins, lo, hi, out=outs)
    assert timing["launches"] == 5
    _assert_route(engine, "bins", "fast" if fast else "ieee", nbins, ranges, 0)
    cast, want = bn.project_cast_hist(x, [0, 1], nbins, lo, hi)
    np.testing.assert_array_equal(counts, want)
    for j in range(2):
        np.testing.assert_array_equal(_bits(outs[j]), _bits(cast[j]), err_msg=f"column {j}")
