"""CPU ORACLE (test infrastructure, NOT product code) — numpy restatement of the benchmark
("B") semantics of the projection -> cast -> histogram path, written independently of
``oracle/bsem.c`` so the two can check each other.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` leg may import this.

Reference sites restated (under /root/reference/microservices):
  * projection  ``projection_image/projection.py:38-43``  — select columns, keep row identity.
  * cast        ``data_type_handler_image/data_type_update.py:40-43`` — value -> number; the
                benchmark's numeric cast is binary64 -> binary32 round-to-nearest-even.
  * histogram   ``histogram_image/histogram.py:31-36``   — ``$group``/``$sum:1`` counts per key;
                B-semantics key = fixed-width bin of the cast value (SURVEY.md §8c);
                for uint8 columns key = value (exactly ``$group``).

PARITY UNPINNED for fp32 cast + binning (the reference defines neither; no upstream tests exist,
SURVEY.md §4).  This module and bsem.c are the definition.
"""
from __future__ import annotations

import numpy as np

CANONICAL_NAN_BITS = np.uint32(0x7FC00000)
SPECIAL_PERIOD = 1009
NUM_SPECIALS = 20
_MASK64 = (1 << 64) - 1


def cast_f64_f32(x: np.ndarray) -> np.ndarray:
    """binary64 -> binary32, round-to-nearest-even; every NaN becomes 0x7fc00000."""
    x = np.asarray(x, dtype=np.float64)
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        f = x.astype(np.float32)
    bits = f.view(np.uint32).copy()
    bits[np.isnan(f)] = CANONICAL_NAN_BITS
    return bits.view(np.float32)


def bin_width(lo, hi, nbins: int) -> np.float32:
    lo32, hi32 = np.float32(lo), np.float32(hi)
    return np.float32(np.float32(hi32 - lo32) / np.float32(nbins))


def bin_index_f32(x: np.ndarray, lo, hi, nbins: int) -> np.ndarray:
    """bin of each fp32 value, -1 where skipped (NaN or outside [lo, hi])."""
    x = np.asarray(x, dtype=np.float32)
    lo32, hi32 = np.float32(lo), np.float32(hi)
    w = bin_width(lo, hi, nbins)
    with np.errstate(invalid="ignore", over="ignore"):
        ok = (x >= lo32) & (x <= hi32)
        d = (x - lo32).astype(np.float32)      # fp32 RN subtract
        t = (d / w).astype(np.float32)         # fp32 RN divide
    idx = np.full(x.shape, -1, dtype=np.int64)
    ti = np.trunc(t[ok]).astype(np.int64)
    idx[ok] = np.minimum(ti, nbins - 1)
    return idx


def auto_range(mins, maxs, nfinite, nbins: int | None = None):
    """Range of an ``nbins``-bin histogram request that carries no ``range`` (SURVEY.md §2.1 C2), per column, from the
    min / max of the finite cast values.  B-semantics, frozen here (the reference defines no bins at all).  Without
    ``nbins`` the last rule (which needs the bin count) is skipped; the result is the same for every column whose
    min and max are at least 2^-133 apart, since no bin count up to LO_MAX_BINS can make their width round to 0:

    * no finite value (empty, all-null or all-NaN/inf column): [0, 1], as ``numpy.histogram`` does for empty input;
    * constant column (min == max): [min - 0.5, max + 0.5] in fp32, again numpy's rule; where +-0.5 is below half an
      ulp (|v| >= 2^24) the edges move to the neighbouring fp32 values instead, so hi > lo always holds; where such a
      neighbour is +-inf (v = +-FLT_MAX) that edge stays at v and the other is the inward neighbour
      (FLT_MAX -> [prev(FLT_MAX), FLT_MAX]: the closed last bin holds v);
    * otherwise [min, max];
    * then, if the fp32 width (hi - lo) / nbins rounds to 0, hi is raised to the smallest fp32 value h for which
      (h - lo) / nbins does not (bins about one subnormal ulp wide, max still inside).
    If hi - lo overflows fp32 the range is left as it is: no finite fp32 range of that width exists, and the histogram
    rejects it."""
    lo = np.array(mins, dtype=np.float32).copy()
    hi = np.array(maxs, dtype=np.float32).copy()
    n = np.asarray(nfinite)
    up, down = np.float32(np.inf), np.float32(-np.inf)
    for j in range(lo.shape[0]):
        if n[j] == 0:
            lo[j], hi[j] = np.float32(0.0), np.float32(1.0)
            continue
        with np.errstate(over="ignore"):
            if lo[j] == hi[j]:
                v = lo[j]
                a, b = np.float32(v - np.float32(0.5)), np.float32(v + np.float32(0.5))
                if a == v:
                    a = np.nextafter(v, down, dtype=np.float32)
                if b == v:
                    b = np.nextafter(v, up, dtype=np.float32)
                if not np.isfinite(b):
                    a, b = np.nextafter(v, down, dtype=np.float32), v
                elif not np.isfinite(a):
                    a, b = v, np.nextafter(v, up, dtype=np.float32)
                lo[j], hi[j] = a, b
            # the first fp32 value above max whose width is positive, one ulp at a time (at most about nbins / 2
            # steps: the width is 0 only while hi - lo <= nbins * 2^-150)
            while nbins is not None and bin_width(lo[j], hi[j], nbins) == 0:
                hi[j] = np.nextafter(hi[j], up, dtype=np.float32)
    return lo, hi


def hist_f32(x: np.ndarray, lo, hi, nbins: int) -> np.ndarray:
    idx = bin_index_f32(x, lo, hi, nbins)
    return np.bincount(idx[idx >= 0], minlength=nbins).astype(np.uint64)


def project_cast_hist(table: np.ndarray, col_idx, nbins: int | None = None, lo=None, hi=None):
    """table: [ncols, nrows] float64 (columnar).  Returns (out [k, nrows] float32, counts [k, nbins] uint64 | None)."""
    table = np.asarray(table, dtype=np.float64)
    col_idx = list(col_idx)
    out = np.empty((len(col_idx), table.shape[1]), dtype=np.float32)
    counts = np.zeros((len(col_idx), nbins), dtype=np.uint64) if nbins else None
    for j, c in enumerate(col_idx):
        out[j] = cast_f64_f32(table[c])
        if nbins:
            counts[j] = hist_f32(out[j], lo[j], hi[j], nbins)
    return out, counts


def hist_u8_cols(table: np.ndarray, col_idx) -> np.ndarray:
    """table: [ncols, nrows] uint8.  counts [k, 256] uint64 — $group value counts of byte columns."""
    table = np.asarray(table, dtype=np.uint8)
    return np.stack([np.bincount(table[c], minlength=256).astype(np.uint64) for c in col_idx])


def checksum(col: np.ndarray, row_offset: int = 0) -> int:
    """sum bits(x[r]) * (2*(row_offset+r)+1) mod 2^64 (bits zero-extended)."""
    col = np.ascontiguousarray(col)
    utype = {8: np.uint64, 4: np.uint32, 1: np.uint8}[col.dtype.itemsize]
    bits = col.view(utype).astype(np.uint64)
    r = np.arange(col.shape[0], dtype=np.uint64) + np.uint64(row_offset)
    with np.errstate(over="ignore"):
        wgt = r * np.uint64(2) + np.uint64(1)
        return int(np.sum(bits * wgt, dtype=np.uint64)) & _MASK64


# ---- counter-based synthetic tables (twin of lo_table_fill_synthetic_dev) ---------------------------
def splitmix64(z: np.ndarray) -> np.ndarray:
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def _u(seed: int, col: int, rows: np.ndarray) -> np.ndarray:
    key = np.uint64((seed ^ (col << 40)) & _MASK64)
    return splitmix64(np.bitwise_xor(rows.astype(np.uint64), key))


def special_values(lo: float, hi: float) -> np.ndarray:
    lo, hi = np.float64(lo), np.float64(hi)
    hi_bits = np.array([hi]).view(np.uint64)[0]
    above = np.array([hi_bits + np.uint64(1) if hi > 0 else hi_bits - np.uint64(1)], dtype=np.uint64).view(np.float64)[0]
    span = hi - lo
    vals = np.array([
        0.0, -0.0, 1e-40, 1e-46, -1e-46, 1e39, -1e39, 0.0, 0.0,
        1.0 + 2.0 ** -24, 1.0 + 3 * 2.0 ** -24, 16777217.0, 3.4028235677973366e38,
        hi, lo, above, hi + span * 2.0 ** -20, lo - span * 2.0 ** -20, np.inf, -np.inf,
    ], dtype=np.float64)
    bits = vals.view(np.uint64)
    bits[7] = np.uint64(0x7FF8000000000000)
    bits[8] = np.uint64(0xFFF4000000000001)
    assert len(vals) == NUM_SPECIALS
    return vals


def synth_f64(kind: int, seed: int, col: int, row0: int, n: int, lo: float = -1000.0, hi: float = 1000.0) -> np.ndarray:
    rows = np.arange(row0, row0 + n, dtype=np.uint64)
    u = _u(seed, col, rows)
    frac = (u >> np.uint64(11)).astype(np.float64) * np.float64(2.0 ** -53)
    span = np.float64(hi) - np.float64(lo)
    x = np.float64(lo) + span * frac          # numpy: one RN multiply then one RN add, never fused
    if kind >= 1:
        hit = (rows % np.uint64(SPECIAL_PERIOD)) == np.uint64(col % SPECIAL_PERIOD)
        if hit.any():
            sp = special_values(lo, hi)
            idx = ((rows[hit] // np.uint64(SPECIAL_PERIOD) + np.uint64(col)) % np.uint64(NUM_SPECIALS)).astype(np.int64)
            xb = x.view(np.uint64)
            xb[hit] = sp.view(np.uint64)[idx]   # copy bit patterns (keeps NaN payloads)
    if kind == 2 and col == 0:
        x[:] = np.float64(lo) + span * np.float64(0.75)
    return x


def synth_u8(seed: int, col: int, row0: int, n: int) -> np.ndarray:
    rows = np.arange(row0, row0 + n, dtype=np.uint64)
    u = _u(seed, col, rows)
    py, px = (col % 784) // 28, (col % 784) % 28
    if not (4 <= py < 24 and 4 <= px < 24):
        return np.zeros(n, dtype=np.uint8)
    v = ((u >> np.uint64(8)) & np.uint64(0xFF)).astype(np.uint8)
    v[(u & np.uint64(0xFF)) < np.uint64(0x99)] = 0
    return v


def synth_table_f64(kind: int, seed: int, ncols: int, row0: int, n: int, lo: float = -1000.0, hi: float = 1000.0) -> np.ndarray:
    return np.stack([synth_f64(kind, seed, c, row0, n, lo, hi) for c in range(ncols)])


def synth_table_u8(seed: int, ncols: int, row0: int, n: int) -> np.ndarray:
    return np.stack([synth_u8(seed, c, row0, n) for c in range(ncols)])
