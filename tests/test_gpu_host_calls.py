"""The lo_host_timing figures of the single-pass host calls, pinned on fixed inputs, and a failed scratch allocation.

Bytes are what each call copies (or, for lo_csv_read_host, has always reported); launches are the kernels the call
enqueues on the path these inputs take.
"""
import ctypes as C

import numpy as np
import pytest

from learningorchestra_b200 import _native as N
from learningorchestra_b200.columnar import pack_cells, pack_number_cells

pytestmark = pytest.mark.gpu

P = C.c_void_p
CARRY_BYTES = 56          # sizeof(lo::csv::Carry): six int64 and two uint32


def _p(a):
    return a.ctypes.data_as(P)


def _assert_timing(t, h2d, d2h, launches, kernel):
    assert (t.h2d_bytes, t.d2h_bytes, t.launches) == (h2d, d2h, launches)
    assert t.total_ms > 0
    assert (t.kernel_ms > 0) if kernel else (t.kernel_ms == 0)


def test_value_counts_timing(engine):
    lib, ctx = engine._lib, engine._ctx
    values = np.arange(1000, dtype=np.float64) % 10
    keys, counts, nd, t = np.zeros(16), np.zeros(16, np.uint64), C.c_int64(), N.HostTiming()
    N.check(lib.lo_value_counts_f64_host(ctx, _p(values), 1000, _p(keys), _p(counts), 16, C.byref(nd), C.byref(t)))
    assert nd.value == 10
    _assert_timing(t, 1000 * 8, 10 * 16 + 8, 2, True)

    chars, offsets = pack_cells(["ab", "c", "", "ab", "c", "ab"])
    rows, counts, nd, t = np.zeros(4, np.int64), np.zeros(4, np.uint64), C.c_int64(), N.HostTiming()
    N.check(lib.lo_value_counts_str_host(ctx, _p(chars), _p(offsets), 6, _p(rows), _p(counts), 4, C.byref(nd),
                                         C.byref(t)))
    assert nd.value == 3
    _assert_timing(t, 8 + 7 * 8, 3 * 16 + 8, 2, True)

    # capacity too small: the call fails, but the number of groups and the timing are reported
    t = N.HostTiming()
    rc = lib.lo_value_counts_f64_host(ctx, _p(values), 1000, _p(keys), _p(counts), 4, C.byref(nd), C.byref(t))
    assert rc == N.LO_ERR_INVALID and b"do not fit" in lib.lo_last_error() and nd.value == 10
    _assert_timing(t, 1000 * 8, 4 * 16 + 8, 2, True)


def test_parse_and_format_timing(engine):
    lib, ctx = engine._lib, engine._ctx
    chars, offsets = pack_number_cells(["1.5", "x", "", "-7", "1e300"])
    values, status, t = np.zeros(5), np.zeros(5, np.uint8), N.HostTiming()
    N.check(lib.lo_parse_number_host(ctx, _p(chars), _p(offsets), 5, _p(values), _p(status), C.byref(t)))
    _assert_timing(t, int(offsets[-1]) + 6 * 8, 5 * 9, 1, True)

    values = np.array([1.5, 0.0, -7.0, 1e300])
    status = np.array([N.LO_NUM_FLOAT, N.LO_NUM_EMPTY, N.LO_NUM_INTEGER, N.LO_NUM_FLOAT], np.uint8)
    timing = {}
    text, offs = engine.format_number_host(values, status, timing)
    assert bytes(text) == b"1.5-71e+300"
    assert (timing["h2d_bytes"], timing["d2h_bytes"], timing["launches"]) == (4 * 9, 5 * 8 + 8 + 11, 3)
    assert timing["kernel_ms"] > 0

    offs, t = np.zeros(5, np.int64), N.HostTiming()            # sizes only: no chars buffer, no text kernel
    N.check(lib.lo_format_number_host(ctx, _p(values), _p(status), 4, _p(offs), None, 0, C.byref(t)))
    assert list(offs) == [0, 3, 3, 5, 11]
    _assert_timing(t, 4 * 9, 5 * 8 + 8, 2, True)


@pytest.mark.parametrize("body, kept, ncols, nchars, launches", [
    (b"a,b\n1,2\n3,4\n", 3, 2, 6, 8),
    (b"a,b\n\x00,5\n", 1, 2, 2, 8),          # the first data row fails: the header is kept
    (b"a\x00,b\n1,2\n", 0, 0, 0, 6),         # the header fails: nothing is kept, no scan and no text kernel
])
def test_csv_timing(engine, body, kept, ncols, nchars, launches):
    lib, ctx = engine._lib, engine._ctx
    buf = np.frombuffer(body, np.uint8)
    h, info, t1, t2 = P(), N.CsvInfo(), N.HostTiming(), N.HostTiming()
    N.check(lib.lo_csv_read_host(ctx, _p(buf), buf.size, C.byref(h), C.byref(info), C.byref(t1)))
    try:
        assert (info.records, info.ncols, info.chars) == (kept, ncols, nchars)
        # d2h: the last carry and summary, the two first failures, then 16 bytes for the text size and the failure
        # key (counted whether or not the text size was read)
        _assert_timing(t1, len(body), 2 * CARRY_BYTES + 16 + 16, launches, True)
        offsets = np.zeros(max(ncols * (kept + 1), 1), np.int64)
        chars = np.zeros(max(nchars, 1), np.uint8)
        N.check(lib.lo_csv_columns_host(h, _p(offsets), _p(chars), chars.size, C.byref(t2)))
        _assert_timing(t2, 0, ncols * (kept + 1) * 8 + nchars, 0, False)
    finally:
        N.check(lib.lo_csv_free(h))


def test_minmax_cast_host_timing(engine):
    lib, ctx = engine._lib, engine._ctx
    cols = [np.linspace(-1.0, 1.0, 5000), np.full(5000, np.nan)]
    in_p = (P * 2)(*[c.ctypes.data for c in cols])
    mins, maxs, cnt, t = np.zeros(2, np.float32), np.zeros(2, np.float32), np.zeros(2, np.uint64), N.HostTiming()
    N.check(lib.lo_minmax_cast_host(ctx, in_p, 5000, 2, _p(mins), _p(maxs), _p(cnt), C.byref(t)))
    assert list(mins) == [-1.0, 0.0] and list(maxs) == [1.0, 0.0] and list(cnt) == [5000, 0]
    _assert_timing(t, 2 * 5000 * 8, 2 * 3 * 8, 1, False)


def test_failed_scratch_allocation_leaves_the_context_usable(engine):
    """A capacity of 2^40 groups asks cudaMallocAsync for 16 TiB of output scratch: an ordinary allocation error the
    runtime returns.  The call fails before it writes any entry, so one-entry host buffers are enough."""
    lib, ctx = engine._lib, engine._ctx
    values = np.arange(100, dtype=np.float64)
    keys, counts, nd = np.zeros(1), np.zeros(1, np.uint64), C.c_int64(-1)
    rc = lib.lo_value_counts_f64_host(ctx, _p(values), 100, _p(keys), _p(counts), 1 << 40, C.byref(nd), None)
    assert rc == N.LO_ERR_NOMEM and lib.lo_last_error().startswith(b"value_counts_f64: ")
    assert nd.value == 0
    keys, counts = engine.value_counts_f64_host(values)
    assert sorted(keys) == list(values) and set(counts) == {1}


def test_project_cast_hist_host_rejects_a_short_out_list(engine):
    cols = [np.zeros(100) for _ in range(3)]
    with pytest.raises(N.LoexecError) as e:
        engine.project_cast_hist_host(cols, 8, -1.0, 1.0, out=[np.zeros(100, np.float32)])
    assert e.value.code == N.LO_ERR_INVALID and "out_cols[1] is NULL" in e.value.message
