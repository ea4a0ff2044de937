"""CPU: the decimal-text -> binary64 parser the GPU kernel runs (csrc/parse_number.cuh, __host__ __device__)
compiled with g++ and checked against CPython's own float() — the reference's cast is literally
``float(document[field])`` followed by ``is_integer()`` (data_type_update.py:40-43)."""
import ctypes as C
import math
import random
import struct
import subprocess
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
SO = ROOT / "tests" / "native" / "_build" / "libparse_harness.so"
FLOAT, INTEGER, EMPTY, INVALID, UNSUPPORTED = 0, 1, 2, 3, 4


@pytest.fixture(scope="module")
def parse():
    src = ROOT / "tests" / "native" / "parse_harness.cpp"
    hdr = ROOT / "learningorchestra_b200" / "csrc" / "parse_number.cuh"
    if not SO.exists() or SO.stat().st_mtime < max(src.stat().st_mtime, hdr.stat().st_mtime):
        SO.parent.mkdir(exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", str(src), "-I",
                        str(ROOT / "learningorchestra_b200" / "csrc"), "-o", str(SO)], check=True)
    lib = C.CDLL(str(SO))

    def run(strings):
        enc = [s.encode("utf-8") if isinstance(s, str) else s for s in strings]
        offs = np.zeros(len(enc) + 1, dtype=np.int64)
        np.cumsum([len(b) for b in enc], out=offs[1:])
        buf = np.frombuffer(b"".join(enc) + b"\0", dtype=np.uint8)
        bits = np.zeros(len(enc), dtype=np.uint64)
        st = np.zeros(len(enc), dtype=np.uint8)
        lib.parse_batch(buf.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p), C.c_int64(len(enc)),
                        bits.ctypes.data_as(C.c_void_p), st.ctypes.data_as(C.c_void_p))
        return bits, st
    return run


def expected(s):
    """(status, bits) per CPython float() + the reference's integer collapse."""
    if s == "":
        return EMPTY, 0
    try:
        v = float(s)
    except ValueError:
        return INVALID, 0
    bits = struct.unpack("<Q", struct.pack("<d", v))[0]
    if math.isnan(v):
        bits = (bits & (1 << 63)) | 0x7FF8000000000000
    return (INTEGER if (math.isfinite(v) and v.is_integer()) else FLOAT), bits


def check(parse, strings):
    bits, st = parse(strings)
    for s, b, t in zip(strings, bits, st):
        es, eb = expected(s)
        assert t == es, (s, int(t), es)
        if es in (FLOAT, INTEGER):
            if math.isnan(struct.unpack("<d", struct.pack("<Q", eb))[0]):
                assert (int(b) & 0x7FFFFFFFFFFFFFFF) == 0x7FF8000000000000, s
            else:
                assert int(b) == eb, (s, hex(int(b)), hex(eb))


# ---- the corpus: one builder per family of cells, shared with the device tests (test_gpu_parse.py) ----------------
def grammar_cases():
    """The reference's cast vectors and the grammar's cases: signs, points, exponents, whitespace, underscores,
    inf / nan spellings, zeros, round-trip and overflow / underflow edges, and a few non-ASCII cells."""
    import json
    vec = json.loads((ROOT / "tests" / "golden" / "reference_cast_vectors.json").read_text())
    cases = [s for s in vec["in"] if s is not None]
    cases += ["1", "-1", "+1", "1.", ".5", "-.5", "+.5e1", "1.e5", ".e5", ".", "", " ", "  7  ", "\t7\n", "\x1c7\x1f", "7 7",
              "1e", "1e+", "1e-", "1e5", "1E5", "1e+05", "1e-05", "1e5.0", "1.5.2", "--1", "+-1", "1-", "abc", "0x10", "1f",
              "inf", "INF", "Infinity", "-infinity", "+inf", "infinit", "infinityy", "in f", "nan", "NaN", "-nan", "+NAN", "nan(1)",
              "1_000", "1__000", "_1", "1_", "1_.5", "1._5", "1.5_5", "1_0.5_0e1_0", "1e_5", "1_e5", "1e5_", "-_1", "+1_0",
              "0", "-0", "0.0", "-0.0", "00", "007", "0e0", "0e999999999", "-0e-999999999", "000.000", "1\x00", "\x001",
              "9007199254740993", "9007199254740992", "9007199254740991", "18014398509481985", "1e22", "1e23", "8.5e22",
              "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308", "1.797693134862315807e308", "1e309", "-1e309",
              "4.9406564584124654e-324", "2.4703282292062327e-324", "2.4703282292062328e-324", "2.47032822920623272e-324", "1e-400",
              "2.2250738585072014e-308", "2.2250738585072011e-308", "2.225073858507201e-308", "1e-323", "3e-324", "2e-324",
              "0.1", "0.2", "0.3", "0.30000000000000004", "123456789012345678", "1234567890123456789", "12345678901234567890",
              "123456789012345678901234567890", "0.000000000000000000000000000001", "1" + "0" * 400, "0." + "0" * 400 + "1",
              "1e99999999999999999999", "1e-99999999999999999999", "１２", "٣", "1 ", "é"]
    return cases


def random_short_decimals():
    """300 000 cells of at most 19 significant digits: repr of random doubles, integers with exponents, fixed-point
    decimals, digit strings with a point anywhere, and small mantissas at the ends of the exponent range."""
    rng = random.Random(20260921)
    cases = []
    for _ in range(300_000):
        kind = rng.random()
        if kind < 0.3:
            s = repr(struct.unpack("<d", struct.pack("<Q", rng.getrandbits(64)))[0])
            if "n" in s:      # nan / inf
                s = repr(rng.uniform(-1e6, 1e6))
        elif kind < 0.5:
            s = f"{rng.randint(0, 10 ** rng.randint(1, 19))}" + ("" if rng.random() < 0.5 else f"e{rng.randint(-330, 310)}")
        elif kind < 0.7:
            s = f"{rng.uniform(-1000, 1000):.{rng.randint(0, 17)}f}"
        elif kind < 0.85:
            d = rng.randint(1, 19)
            digits = "".join(rng.choice("0123456789") for _ in range(d))
            pos = rng.randint(0, d)
            s = rng.choice(["", "-", "+"]) + digits[:pos] + "." + digits[pos:] + rng.choice(["", f"e{rng.randint(-340, 308)}", f"E+{rng.randint(0, 300)}"])
        else:
            s = f"{rng.randint(1, 999)}e{rng.randint(-345, 310)}"
        cases.append(s)
    return cases


def halfway_and_long_digits():
    """> 19 significant digits: exact midpoints between adjacent doubles (ties-to-even), and midpoints nudged by
    one unit hundreds of digits further right (must go up / down) — the big-integer slow path — then 20 000 random
    strings of 20 to 60 digits."""
    rng = random.Random(7)
    cases = []
    for _ in range(3000):
        e = rng.choice([rng.randint(-1074, -1000), rng.randint(-60, 60), rng.randint(900, 970), rng.randint(-1022, 1023) - 52])
        m = rng.getrandbits(53) | (1 << 52) if e > -1074 else rng.getrandbits(52) | 1
        lo = Fraction(m) * Fraction(2) ** e
        mid = lo + Fraction(2) ** (e - 1)
        # exact decimal expansion of mid (denominator is a power of two)
        num, den = mid.numerator, mid.denominator
        k = den.bit_length() - 1
        digits = str(num * 5 ** k)
        s = digits if k == 0 else (digits[:-k] or "0") + "." + digits[-k:].rjust(k, "0") if len(digits) > k else "0." + digits.rjust(k, "0")
        if len(s) > 1000:
            continue
        cases.append(s)
        cases.append(s + "1" if "." in s else s + ".0000000001")
        if s.rstrip("0") != s and "." in s:
            cases.append(s.rstrip("0"))
        # one unit below in the last place
        t = list(s)
        for i in range(len(t) - 1, -1, -1):
            if t[i].isdigit() and t[i] != "0":
                t[i] = str(int(t[i]) - 1)
                break
        cases.append("".join(t) + "9" * 30)
    for _ in range(20000):
        d = rng.randint(20, 60)
        digits = "".join(rng.choice("0123456789") for _ in range(d))
        pos = rng.randint(0, d)
        cases.append(digits[:pos] + "." + digits[pos:] + rng.choice(["", f"e{rng.randint(-340, 300)}"]))
    return cases


def long_cells():
    """Cells of thousands of bytes: digits past the 800th only matter as a sticky bit."""
    return ["1" * 1025, "0" * 5000 + "7", "1" * 400 + "." + "9" * 3000, "0." + "0" * 2000 + "123", "9" * 309, "9" * 308 + "." + "5" * 2000,
            "2.4703282292062327208051355972538996e-324" + "0" * 1500 + "1", " " * 1500 + "1e5" + "\t" * 900,
            "1" + "_0" * 700, "4.9e-324" + "0" * 2000, "1" + "0" * 1100 + "e-1100", "0" * 3000, "." + "0" * 3000 + "e5"]


def unicode_cells():
    """Unicode decimal digits and whitespace, which float(str) maps to ASCII first, and characters it refuses."""
    return ["１２", "٣.٥", "\u2003 5\u00a0", "１_０", "-１e２", "é1", "1é", "１٣.５e-１", "\u30001\u3000", "१२३", "1\u00b2", "½", "\x1c5", "5\x85"]


def test_grammar_and_reference_cast_vectors(parse):
    cases = grammar_cases()
    from learningorchestra_b200.columnar import ascii_number_text
    bits, st = parse(cases)
    for s, b, t in zip(cases, bits, st):
        assert t == UNSUPPORTED if any(ord(ch) >= 0x80 for ch in s) else t != UNSUPPORTED, s   # raw UTF-8 is reported, not guessed
    # ... and through the packer's normalisation (what float(str) does first) every case is decided as CPython decides it
    bits, st = parse([ascii_number_text(c) for c in cases])
    for s, b, t in zip(cases, bits, st):
        es, eb = expected(s)
        assert t == es, (repr(s), int(t), es)
        if es in (FLOAT, INTEGER) and not math.isnan(struct.unpack("<d", struct.pack("<Q", eb))[0]):
            assert int(b) == eb, (s, hex(int(b)), hex(eb))


def test_random_short_decimals(parse):
    check(parse, random_short_decimals())


def test_halfway_and_long_digit_strings(parse):
    """> 19 significant digits: exact midpoints between adjacent doubles (ties-to-even), and midpoints nudged by
    one unit hundreds of digits further right (must go up / down) — the big-integer slow path."""
    check(parse, halfway_and_long_digits())


def test_long_cells_and_unicode_text(parse):
    """No length limit short of 1 MiB: digits past the 800th only matter as a sticky bit.  Unicode decimal digits and
    whitespace go through the packer's float(str) normalisation."""
    from learningorchestra_b200.columnar import ascii_number_text
    check(parse, long_cells())
    uni = unicode_cells()
    bits, st = parse([ascii_number_text(c) for c in uni])
    for s, b, t in zip(uni, bits, st):
        es, eb = expected(s)
        assert t == es, (repr(s), int(t), es)
        if es in (FLOAT, INTEGER):
            assert int(b) == eb, (s, hex(int(b)), hex(eb))
    bits, st = parse(["é1", b"\xff", "1" * ((1 << 20) + 1)])
    assert st.tolist() == [UNSUPPORTED, UNSUPPORTED, UNSUPPORTED]
