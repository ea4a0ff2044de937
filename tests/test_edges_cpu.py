"""CPU: the bin-edge tables of the fused tile kernel and the shape of its steady-state loop.

The host computes, per histogram column, the edges E[i] = the smallest fp32 value whose bin is >= i; the EDGES kernels
bin with one table lookup and one comparison.  Here the edges are checked against the oracle's binning, and the SASS of
the shipped kernel is counted: the per-element work of the hot loop is what the histogram costs in power."""
import ctypes
import json
import re
import subprocess
from collections import Counter
from pathlib import Path

import numpy as np
import pytest

from oracle import bsem_numpy as bn
from test_gpu_hist_routes import EDGE_RANGES

ROOT = Path(__file__).resolve().parent.parent
KAT = json.loads((ROOT / "tests" / "golden" / "bin_kat.json").read_text())["cases"]

# the ranges the exhaustive GPU self-tests run, plus a divisor with an all-ones significand and extreme widths
TRIPLES = [
    (-1000.0, 1000.0, 256), (-1000.0, 1000.0, 10), (0.0, 1.0, 256), (0.0, 255.0, 255), (-3.0, 7.0, 3),
    (1e-30, 2e-30, 100), (-1e30, 1e30, 256), (0.1, 0.7, 7), (-123.456, 789.012, 177), (5.0, 5.000001, 2),
    (0.0, 512.0, 256), (-1.0, 80.0, 10),
    (0.0, float(np.float32(np.uint32(0x3FFFFFFF).view(np.float32)) * np.float32(4)), 4),
    (0.0, 1e-37, 8), (-1e38, 1e38, 2), (1e6, 1e6 + 64.0, 256), (-1.5e38, 1.5e38, 256),
    (0.0, 2.0 ** -92, 256), (0.0, 2.0 ** 108, 256), (-(2.0 ** 107), 2.0 ** 107, 256),     # w = 2^-100, 2^100: the window's ends
]


def _edges(lo, hi, nbins):
    from learningorchestra_b200 import _native
    lib = _native.load()
    out = np.zeros(nbins + 1, np.float32)
    rc = lib.lo_hist_edges(ctypes.c_float(lo), ctypes.c_float(hi), nbins, out.ctypes.data_as(ctypes.c_void_p))
    assert rc == _native.LO_OK
    return out


def _check_edges(lo, hi, nbins, extra=()):
    lo32, hi32 = np.float32(lo), np.float32(hi)
    E = _edges(lo, hi, nbins)
    assert E[0] == lo32 and E[nbins] == np.nextafter(hi32, np.float32(np.inf))
    assert np.all(np.diff(E) >= 0)
    inner = E[1:nbins]
    if nbins > 1:
        # each edge is in range, is binned at or above its index, and its predecessor (if still >= lo) below it
        ok = inner <= hi32
        assert np.all(bn.bin_index_f32(inner[ok], lo, hi, nbins) >= np.arange(1, nbins)[ok])
        prev = np.nextafter(inner, np.float32(-np.inf))
        inrange = ok & (prev >= lo32)
        assert np.all(bn.bin_index_f32(prev[inrange], lo, hi, nbins) < np.arange(1, nbins)[inrange])
    # binning by the edges equals the oracle on the edges, their neighbours, the range ends and any extra values
    x = np.concatenate([E, np.nextafter(E, np.float32(-np.inf)), np.nextafter(E, np.float32(np.inf)),
                        np.array([lo32, hi32], np.float32), np.asarray(extra, np.float32)]).astype(np.float32)
    x = x[np.isfinite(x)]
    want = bn.bin_index_f32(x, lo, hi, nbins)
    got = np.searchsorted(inner, x, side="right")
    got = np.where((x >= lo32) & (x <= hi32), got, -1)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("case", range(len(KAT)))
def test_edges_bin_the_kat_vectors_like_the_oracle(built, case):
    c = KAT[case]
    _check_edges(c["lo"], c["hi"], c["nbins"], extra=c["x"])
    E = _edges(c["lo"], c["hi"], c["nbins"])
    x = np.asarray(c["x"], np.float32)
    got = np.where((x >= np.float32(c["lo"])) & (x <= np.float32(c["hi"])), np.searchsorted(E[1:c["nbins"]], x, side="right"), -1)
    np.testing.assert_array_equal(got, np.asarray(c["bin"]))


@pytest.mark.parametrize("lo,hi,nbins", TRIPLES + [r for r in EDGE_RANGES if r not in TRIPLES])
def test_edges_of_the_self_test_ranges(built, lo, hi, nbins):
    """The ranges of the exhaustive self-tests and of the GPU route tests (up to 65 536 bins), whose values are placed
    on and around these edges."""
    rng = np.random.default_rng(nbins)
    _check_edges(lo, hi, nbins, extra=rng.uniform(lo, hi, 20_000))


def test_edges_of_random_ranges(built):
    rng = np.random.default_rng(20261015)
    for _ in range(300):
        scale = 10.0 ** rng.uniform(-30, 30)
        a, b = np.sort(rng.uniform(-1, 1, 2) * scale)
        if rng.random() < 0.3:
            b = a + abs(a) * 10.0 ** rng.uniform(-7, -2) + 1e-38
        lo, hi = np.float32(a), np.float32(b)
        nbins = int(rng.integers(1, 257))
        w = bn.bin_width(lo, hi, nbins)
        if not (hi > lo and np.isfinite(w) and w > 0):
            continue
        _check_edges(float(lo), float(hi), nbins, extra=rng.uniform(lo, hi, 2_000))


def _functions(sass):
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2).strip()))
    return out


def _streaming_loop(ins):
    """Body of the largest backward branch that converts fp64 -> fp32: the full-tile steady state."""
    best = []
    for addr, txt in ins:
        m = re.search(r"\bBRA\b.*?(0x[0-9a-f]+)", txt)
        if m and int(m.group(1), 16) < addr:
            body = [t for a, t in ins if int(m.group(1), 16) <= a <= addr]
            if any("F2F.F32.F64" in t for t in body) and len(body) > len(best):
                best = body
    return best


def test_fused_kernel_loop_instruction_budget(built):
    from learningorchestra_b200 import _native
    sass = subprocess.run(["cuobjdump", "-sass", str(_native.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    fns = _functions(sass)
    per_elem = {}
    for name, ins in fns.items():
        m = re.match(r"_ZN2lo19k_project_cast_histILi(\d)ELb(\d)ELb1ELb(\d)EEE", name)
        if not m or (m.group(2) == "0" and m.group(1) != "1"):      # an f64 copy converts nothing
            continue
        body = _streaming_loop(ins)
        elems = sum("F2F.F32.F64" in t for t in body)
        assert elems > 0, name
        per_elem[m.groups()] = len(body) / elems
        if m.group(2) == "1" and m.group(3) == "1":
            ops = Counter(re.sub(r"^@!?U?P\w+\s+", "", t).split()[0] for t in body)
            assert not any(op.startswith("IMAD.MOV") for op in ops), (name, ops)
            assert ops["LDS.128"] == elems and ops["LDS.U8"] == elems and ops["STS.U8"] == elems, ops
    assert per_elem[("1", "1", "1")] <= 16.0, per_elem          # the S100 kernel (cast-only: see below)
    assert per_elem[("1", "0", "0")] <= 5.0, per_elem
    for out in "012":
        assert per_elem[(out, "1", "1")] <= 16.0, per_elem


def test_fused_kernels_have_no_stack_frame(built):
    from learningorchestra_b200 import _native
    res = subprocess.run(["cuobjdump", "-res-usage", str(_native.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    seen = 0
    lines = res.splitlines()
    for i, line in enumerate(lines):
        if re.search(r"Function _ZN2lo19k_project_cast_histILi\dELb1ELb1ELb\dEEE", line):
            assert "STACK:0 " in lines[i + 1], (line, lines[i + 1])
            seen += 1
    assert seen == 6
