"""CPU: the pieces behind the GPU group-by and the range pre-pass that can be checked without a GPU.

* The hashes of the group-by kernels (``hash_bytes``, ``splitmix64`` in csrc/kernels.cuh, both ``__host__ __device__``)
  compiled with nvcc into a host harness, against the numpy ports the GPU tests use to build adversarial inputs and
  against the committed collision pairs (tests/golden/hash_collisions.json).  Without this a wrong port would make those
  GPU tests pass without exercising what they claim.
* ``auto_range`` (product: ``columnar``; definition: ``oracle.bsem_numpy``) on the columns whose plain min / max are not
  a range the histogram accepts, and the agreement of the two functions.
"""
import ctypes as C
import importlib.util
import json
import subprocess
from pathlib import Path

import numpy as np
import pytest

from learningorchestra_b200 import columnar
from oracle import bsem_numpy as bn

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden"
F32_MAX = np.finfo(np.float32).max
TINY = np.float32(2.0 ** -149)                 # the smallest fp32 subnormal


def _collision_module():
    spec = importlib.util.spec_from_file_location("make_hash_collisions", GOLD / "make_hash_collisions.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def hashlib_native(tmp_path_factory):
    from learningorchestra_b200.build import _nvcc
    so = tmp_path_factory.mktemp("hash_harness") / "libhash_harness.so"
    # PTX only: the harness calls the host copies; nothing device-side is run or needs machine code
    subprocess.run([_nvcc(), "-gencode", "arch=compute_90a,code=compute_90a", "-std=c++17", "-Xcompiler", "-fPIC",
                    "-shared", "-I", str(ROOT / "include"), "-I", str(ROOT / "learningorchestra_b200" / "csrc"),
                    "-o", str(so), str(ROOT / "tests" / "native" / "hash_harness.cu")], check=True)
    lib = C.CDLL(str(so))

    def hash_cells(cells):
        enc = [c if isinstance(c, bytes) else c.encode() for c in cells]
        offsets = np.zeros(len(enc) + 1, dtype=np.int64)
        np.cumsum([len(b) for b in enc], out=offsets[1:])
        chars = np.frombuffer(b"".join(enc) + b"\0", dtype=np.uint8)
        out = np.zeros(len(enc), dtype=np.uint64)
        lib.hash_cells(chars.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), C.c_int64(len(enc)),
                       out.ctypes.data_as(C.c_void_p))
        return out

    def splitmix64(z):
        z = np.ascontiguousarray(z, dtype=np.uint64)
        out = np.zeros_like(z)
        lib.splitmix64_batch(z.ctypes.data_as(C.c_void_p), C.c_int64(z.size), out.ctypes.data_as(C.c_void_p))
        return out
    return hash_cells, splitmix64


def test_collision_fixture_matches_the_kernels_hash(hashlib_native):
    hash_cells, splitmix64 = hashlib_native
    fx = json.loads((GOLD / "hash_collisions.json").read_text())
    mask, shift = np.uint64(fx["table_slots"] - 1), np.uint64(fx["tag_shift"])
    assert fx["table_slots"] == 1024 and fx["tag_shift"] == 31 and len(fx["pairs"]) >= 3
    for p in fx["pairs"]:
        assert p["a"] != p["b"] and len(p["a"]) == len(p["b"]) == fx["length"]
        ha, hb = hash_cells([p["a"], p["b"]])
        assert (f"{int(ha):016x}", f"{int(hb):016x}") == (p["hash_a"], p["hash_b"])
        assert ha != hb                                                       # different full hashes: the warp
        assert ha >> shift == hb >> shift == np.uint64(int(p["tag"], 16))     # does not merge them, the tag matches
        sa, sb = splitmix64(np.array([ha, hb])) & mask
        assert sa == sb == p["slot"]                                          # and both probe the same start slot


def test_numpy_hash_ports_equal_the_kernels_hash(hashlib_native):
    hash_cells, splitmix64 = hashlib_native
    mod = _collision_module()
    rng = np.random.default_rng(3)
    for length in (0, 1, 7, 8, 33):
        cells = rng.integers(0, 256, (500, length), dtype=np.uint8)
        np.testing.assert_array_equal(mod.hash_bytes(cells), hash_cells([c.tobytes() for c in cells]))
    z = rng.integers(0, 2 ** 64, 100_000, dtype=np.uint64, endpoint=False)
    z[:4] = [0, 1, 2 ** 64 - 1, 0x7FF8000000000000]
    np.testing.assert_array_equal(bn.splitmix64(z), splitmix64(z))          # the GPU tests' probe-slot port
    np.testing.assert_array_equal(mod.splitmix64(z), splitmix64(z))


# ---- auto_range ---------------------------------------------------------------------------------------------------
def _usable(lo, hi, nbins):
    """What lo_project_cast_hist accepts (check_spec): finite edges, hi > lo, a finite positive fp32 width."""
    with np.errstate(over="ignore"):
        w = bn.bin_width(lo, hi, nbins)
    return bool(np.isfinite(lo) and np.isfinite(hi) and hi > lo and np.isfinite(w) and w > 0)


def _both(values, nbins):
    """auto_range of one column of fp64 values through the product and the oracle, from the exact pre-pass results."""
    f = bn.cast_f64_f32(np.asarray(values, dtype=np.float64))
    fin = f[np.isfinite(f)]
    args = ([fin.min()] if fin.size else [0.0], [fin.max()] if fin.size else [0.0], [fin.size], nbins)
    with np.errstate(over="ignore"):
        p, o = columnar.auto_range(*args), bn.auto_range(*args)
    assert p[0].view(np.uint32)[0] == o[0].view(np.uint32)[0] and p[1].view(np.uint32)[0] == o[1].view(np.uint32)[0], (p, o)
    return np.float32(o[0][0]), np.float32(o[1][0]), fin


@pytest.mark.parametrize("values, nbins, lo, hi", [
    ([0.0, 1e-45], 10, 0.0, 6 * 2.0 ** -149),            # width > 0 needs hi - lo > 10 * 2^-150
    ([0.0, 1e-44], 256, 0.0, 129 * 2.0 ** -149),         # 1e-44 casts to 7 * 2^-149
    ([0.0, 1e-45], 65536, 0.0, 32769 * 2.0 ** -149),
    ([-1e-45, 1e-45], 3, -(2.0 ** -149), 2.0 ** -149),    # already usable: unchanged
    ([2.0 ** -125, 2.0 ** -125 + 2.0 ** -148], 7, 2.0 ** -125, 2.0 ** -125 + 2.0 ** -147),   # normal lo, odd nbins
    ([-(2.0 ** -126), -(2.0 ** -126) + 2.0 ** -149], 5, -(2.0 ** -126), -(2.0 ** -126) + 3 * 2.0 ** -149),
    ([float(F32_MAX)] * 3, 10, float(np.nextafter(F32_MAX, np.float32(0))), float(F32_MAX)),
    ([-float(F32_MAX)] * 3, 10, -float(F32_MAX), -float(np.nextafter(F32_MAX, np.float32(0)))),
    ([3.4028235677973366e38, float(F32_MAX)], 10, float(np.nextafter(F32_MAX, np.float32(0))), float(F32_MAX)),
    ([7.0, 7.0], 10, 6.5, 7.5),
    ([2.0 ** 30] * 2, 4, 2.0 ** 30 - 64, 2.0 ** 30 + 128),
    ([np.nan, np.inf, -np.inf], 10, 0.0, 1.0),
    ([1e-46, -1e-46], 10, -0.5, 0.5),                    # both cast to +-0: a constant zero column
])
def test_auto_range_gives_a_usable_range(values, nbins, lo, hi):
    got_lo, got_hi, fin = _both(values, nbins)
    assert (float(got_lo), float(got_hi)) == (lo, hi)
    assert _usable(got_lo, got_hi, nbins)
    if fin.size:
        assert got_lo <= fin.min() and fin.max() <= got_hi                 # every finite value is counted
        assert bn.hist_f32(fin, got_lo, got_hi, nbins).sum() == fin.size
    if fin.size and fin.min() != fin.max() and bn.bin_width(fin.min(), fin.max(), nbins) == 0:
        # the smallest such hi: one fp32 step down the width is 0 again
        assert bn.bin_width(got_lo, np.nextafter(got_hi, np.float32(-np.inf)), nbins) == 0


def test_auto_range_keeps_a_span_that_overflows_fp32():
    """{-3e38, 3e38}: hi - lo overflows fp32 and the binning formula is frozen, so no usable range of that width
    exists; [min, max] is returned and the histogram call rejects it."""
    lo, hi, _ = _both([-3e38, 0.0, 3e38], 10)
    assert (lo, hi) == (np.float32(-3e38), np.float32(3e38))
    assert not _usable(lo, hi, 10)


def test_oracle_auto_range_without_nbins_skips_only_the_width_rule():
    """The oracle's three-argument form (no bin count) gives the same range as any bin count where min and max are at
    least 2^-133 apart, and keeps the constant-column rules; only the subnormal-width rule needs ``nbins``."""
    cases = [([-3.5], [7.25], [9]), ([2.0 ** -133], [2.0 ** -132], [2]), ([F32_MAX], [F32_MAX], [1]),
             ([-F32_MAX], [-F32_MAX], [4]), ([7.0], [7.0], [3]), ([0.0], [0.0], [0])]
    for mins, maxs, nf in cases:
        lo3, hi3 = bn.auto_range(mins, maxs, nf)
        for nbins in (1, 10, 65536):
            lo4, hi4 = bn.auto_range(mins, maxs, nf, nbins)
            assert lo3.view(np.uint32)[0] == lo4.view(np.uint32)[0] and hi3.view(np.uint32)[0] == hi4.view(np.uint32)[0]
    lo, hi = bn.auto_range([0.0], [TINY], [2])
    assert (float(lo[0]), float(hi[0])) == (0.0, 2.0 ** -149)


def test_auto_range_product_and_oracle_agree_on_random_columns():
    rng = np.random.default_rng(8)
    scales = [2.0 ** -149, 2.0 ** -140, 2.0 ** -126, 1e-30, 1.0, 1e30, 3e38]
    for _ in range(400):
        s = scales[rng.integers(len(scales))]
        n = int(rng.integers(1, 5))
        vals = rng.integers(-8, 9, n) * s * rng.choice([1.0, 1.5, 3.0])
        nbins = int(rng.choice([1, 2, 3, 7, 10, 255, 256, 1000, 65536]))
        lo, hi, fin = _both(vals, nbins)
        with np.errstate(over="ignore"):
            if fin.size and not np.isfinite(fin.max() - fin.min()):
                continue
        assert _usable(lo, hi, nbins), (vals, nbins, lo, hi)
