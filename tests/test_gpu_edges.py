"""GPU: the edge-table binning of the fused tile kernel equals the IEEE-divide bin for every fp32 bit pattern, and the
kernels that use it count values at and around every edge exactly like the oracle."""
import numpy as np
import pytest

from oracle import bsem_numpy as bn

pytestmark = pytest.mark.gpu

W_MARKSTEIN = float(np.float32(np.uint32(0x3FFFFFFF).view(np.float32)) * np.float32(4))   # w = 1.9999999: all-ones significand

RANGES = [
    (-1000.0, 1000.0, 256), (-1000.0, 1000.0, 10), (0.0, 1.0, 256), (0.0, 255.0, 255), (-3.0, 7.0, 3),
    (-1e30, 1e30, 256), (0.1, 0.7, 7), (-123.456, 789.012, 177), (5.0, 5.000001, 2),
    (0.0, 512.0, 256), (-1.0, 80.0, 10),
    (0.0, W_MARKSTEIN, 4), (1e6, 1e6 + 64.0, 256), (-1e20, 1e20, 1), (1e-20, 1.5e-20, 256),
    # widths at the ends of the window edges_ok admits (r and r * 2^-9 just normal): w = 2^-100 and w = 2^100
    (0.0, 2.0 ** -92, 256), (0.0, 2.0 ** 108, 256), (-(2.0 ** 107), 2.0 ** 107, 256), (1.0, 1.0 + 2.0 ** -23, 1),
]


@pytest.mark.parametrize("lo,hi,nbins", RANGES)
def test_edge_binning_is_ieee_divide_exhaustively(engine, lo, hi, nbins):
    """All 2^32 fp32 bit patterns: the edge-table counter is the IEEE-divide bin's, or the trash counter where that
    skips the value (NaN, outside [lo, hi])."""
    used, bad = engine.selftest_edges(lo, hi, nbins)
    assert used
    assert bad == 0


def test_widths_outside_the_exponent_window_take_the_ieee_kernel(engine):
    for lo, hi, nbins in [(0.0, 1e-37, 8), (-1e38, 1e38, 2), (1e-30, 2e-30, 100), (0.0, 2.0 ** -93, 256),
                          (0.0, 2.0 ** 108, 128)]:      # w = 2^-101 and w = 2^101, one step outside the window
        used, _ = engine.selftest_edges(lo, hi, nbins)
        assert not used


@pytest.mark.parametrize("lo,hi,nbins", [(-1000.0, 1000.0, 256), (5.0, 5.000001, 2), (0.0, W_MARKSTEIN, 4),
                                         (-123.456, 789.012, 177), (1e6, 1e6 + 64.0, 256)])
def test_values_at_every_edge_count_like_the_oracle(engine, lo, hi, nbins):
    from learningorchestra_b200 import _native
    import ctypes
    E = np.zeros(nbins + 1, np.float32)
    assert _native.load().lo_hist_edges(ctypes.c_float(lo), ctypes.c_float(hi), nbins, E.ctypes.data_as(ctypes.c_void_p)) == 0
    x32 = np.concatenate([E, np.nextafter(E, np.float32(-np.inf)), np.nextafter(E, np.float32(np.inf)),
                          np.array([np.nan, np.inf, -np.inf, 0.0, -0.0], np.float32)])
    rng = np.random.default_rng(nbins)
    x = np.concatenate([np.repeat(x32.astype(np.float64), 7), rng.uniform(lo, hi, 300_000)])
    x = np.concatenate([x, x[::-1]])                 # full tiles (the streaming loop) and a ragged last tile
    x = np.tile(x, 1 + 200_000 // x.size)
    t = engine.table_from_numpy(x[None, :])
    got = engine.project_cast_hist(t, [0], nbins, lo, hi).to_numpy()
    _, exp = bn.project_cast_hist(x[None, :], [0], nbins, [lo], [hi])
    np.testing.assert_array_equal(got, exp)
    t.free()


def test_many_ranges_keep_the_edge_kernel_and_bounded_tables(engine):
    """A service passes a new (lo, hi) with nearly every request.  Thirty distinct ranges, launched on two streams without
    waiting in between, so tables are retired while launches that read them are still queued: every count is the
    oracle's, every launch bins from an edge table (none falls back to the divide) and the cache stays at its bound."""
    import torch
    rng = np.random.default_rng(11)
    rows = 1_000_003
    x = np.stack([rng.uniform(-1500.0, 1500.0, rows), rng.normal(0.0, 300.0, rows)])
    t = engine.table_from_numpy(x)
    _, _, divide0 = engine.edge_tables_info()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    specs, got = [], []
    for i in range(30):
        lo = np.array([-1000.0 - 7.25 * i, -900.0 + i], np.float32)
        hi = np.array([1000.0 + 3.5 * i, 800.0 - 2.0 * i], np.float32)
        nbins = 256 if i % 3 else 10 + i
        if i % 4 == 3:                                      # a range seen before comes back
            lo, hi, nbins = specs[i - 2]
        specs.append((lo, hi, nbins))
        got.append(engine.project_cast_hist(t, [0, 1], nbins, lo, hi, stream=streams[i % 2]))
        tables, nbytes, divide = engine.edge_tables_info()
        assert 1 <= tables <= 8 and nbytes <= 8 * 2 * 257 * 4
        assert divide == divide0
    torch.cuda.synchronize()
    for (lo, hi, nbins), c in zip(specs, got):
        _, exp = bn.project_cast_hist(x, [0, 1], nbins, lo, hi)
        np.testing.assert_array_equal(c.to_numpy(), exp)
    t.free()
