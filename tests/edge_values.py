"""Values at the edges of the binned histogram and of the range pre-pass, and plain references for them.

Shared by the single-device route tests (``test_gpu_hist_routes.py``), the pre-pass tests
(``test_gpu_groupby_prepass.py``) and the multi-GPU group tests (``test_gpu_group_routes.py``).  Every builder is
deterministic, so each rank of a group rebuilds the same columns on its own."""
import ctypes

import numpy as np

from oracle import bsem_numpy as bn

F32_MAX = 3.4028234663852886e38
NAN_BITS = [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFF0000000000001, 0x7FF4000000000000,
            0x7FFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF, 0x7FF8DEADBEEF0001, 0xFFF00000DEADBEEF, 0x7FFC000000000123]


def f64(bits):
    return np.array(bits, dtype=np.uint64).view(np.float64)


F32_MAX_TIE = float(np.float64(np.finfo(np.float32).max) + 2.0 ** 103)    # halfway to 2^128: rounds to +inf
SPECIALS = np.concatenate([
    [0.0, -0.0],
    np.array([1, 3, 0x7FFFFF, 0x80000001, 0x80400000], np.uint32).view(np.float32).astype(np.float64),   # fp32 subnormals
    # overflow in fp32 (the tie at FLT_MAX rounds to inf, one ulp below it to FLT_MAX) and underflow (2^-150 is the tie
    # with 0, 3 * 2^-150 the tie between the two smallest subnormals)
    [F32_MAX_TIE, -F32_MAX_TIE, np.nextafter(F32_MAX_TIE, 0.0), 1e39, -1e300, 2.0 ** -150, -(2.0 ** -150), 3 * 2.0 ** -150,
     1e-46, -1e-300, np.inf, -np.inf],
    f64([0x7FF8000000000000, 0xFFF4000000000001]),      # quiet NaN; negative signalling NaN with a payload
])


def edges(lo, hi, nbins):
    """The bin edges the library bins against (``lo_hist_edges``), as fp32."""
    from learningorchestra_b200 import _native
    E = np.zeros(nbins + 1, np.float32)
    assert _native.load().lo_hist_edges(ctypes.c_float(lo), ctypes.c_float(hi), nbins,
                                        E.ctypes.data_as(ctypes.c_void_p)) == _native.LO_OK
    return E


_columns_cache = {}


def edge_column(lo, hi, nbins):
    """fp64 values on every edge of (lo, hi, nbins) and on both fp32 neighbours, the exact midpoints between an edge and
    each neighbour (round-to-nearest-even ties of the cast) and one fp64 ulp either side of them, the range ends and
    their outer neighbours, special values and a uniform fill; shuffled with a fixed seed."""
    key = (lo, hi, nbins)
    if key not in _columns_cache:
        E = edges(lo, hi, nbins)
        e = E.astype(np.float64)
        up = np.nextafter(E, np.float32(np.inf)).astype(np.float64)
        down = np.nextafter(E, np.float32(-np.inf)).astype(np.float64)
        mids = np.concatenate([(e + up) / 2, (e + down) / 2])       # exact: 25 significant bits
        mids = mids[np.isfinite(mids)]
        lo32, hi32 = np.float32(lo), np.float32(hi)
        ends = np.array([lo32, hi32, np.nextafter(lo32, np.float32(-np.inf)), np.nextafter(hi32, np.float32(np.inf))],
                        np.float64)
        rng = np.random.default_rng(nbins)
        x = np.concatenate([e, up, down, mids, np.nextafter(mids, -np.inf), np.nextafter(mids, np.inf), ends, SPECIALS,
                            rng.uniform(lo, hi, 4096 + nbins)])
        _columns_cache[key] = x[rng.permutation(x.size)]
    return _columns_cache[key]


def prepass_columns(n):
    """Columns of n rows where a min / max / finite-count reduction of the fp32-cast values goes wrong: all NaN (many
    payloads), all +-inf, only values that cast to FLT_MAX, negatives only, +0.0 and -0.0, values that cast to +-0 or
    subnormals, one finite value (first, last, middle row), and normal values."""
    rng = np.random.default_rng(31)
    cols = []
    cols.append(f64(np.array(NAN_BITS, np.uint64)[rng.integers(0, len(NAN_BITS), n)]))             # all NaN
    cols.append(np.where(rng.random(n) < 0.5, np.inf, -np.inf))                                     # all +-inf
    c = np.array([3.4028235677973366e38, 1e39, -1e39, F32_MAX])[rng.integers(0, 4, n)]               # only FLT_MAX
    cols.append(c)                                                                                   # survives the cast
    cols.append(-rng.uniform(1.0, 1e6, n))                                                          # negatives only
    cols.append(np.where(rng.random(n) < 0.5, 0.0, -0.0))                                           # +0.0 and -0.0
    tiny = np.array([1e-46, -1e-46, 1e-40, -1e-40, 2.0 ** -149, 2.0 ** -150, 2.0 ** -150 + 2.0 ** -200, -(2.0 ** -150)])
    c = np.concatenate([tiny, rng.uniform(-1.2e-38, 1.2e-38, n - tiny.size)])                       # -> +-0 / subnormal
    cols.append(c)
    for where in (0, n - 1, n // 2 + 7):                                                            # one finite value
        c = np.full(n, np.nan)
        c[where] = -12.375
        cols.append(c)
    cols.append(rng.normal(0.0, 1e4, n))
    return cols


def ref_minmax(col):
    """(min, max, nfinite) of the finite fp32-cast values; -0.0 orders below +0.0; no finite value -> (0, 0, 0)."""
    f = bn.cast_f64_f32(col)
    fin = f[np.isfinite(f)]
    if fin.size == 0:
        return np.float32(0.0), np.float32(0.0), 0
    mn, mx = fin.min(), fin.max()
    zeros = fin[fin == 0]
    if mn == 0:
        mn = np.float32(-0.0) if np.signbit(zeros).any() else np.float32(0.0)
    if mx == 0:
        mx = np.float32(0.0) if (~np.signbit(zeros)).any() else np.float32(-0.0)
    return mn, mx, fin.size
