"""CPU: the binary64 -> text formatter the GPU kernels run (csrc/format_number.cuh, __host__ __device__) compiled with
g++ and checked byte for byte against CPython's own repr(float) and str(int) — the reference's "string" cast is
literally ``"" if v is None else str(v)`` (data_type_update.py:22-28) — plus the routing of that cast in ``DataType``
(which cells go to the formatter, how the result is stored) with a stand-in engine whose formatter is Python itself."""
import ctypes as C
import json
import math
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

from learningorchestra_b200 import utils
from learningorchestra_b200.column_store import ColumnarDatabase, NumberColumn, TextColumn
from learningorchestra_b200.data_type_update import DataType
from oracle import rsem
from oracle_engine import OracleEngine

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden"
FLOAT, INTEGER, EMPTY = 0, 1, 2


@pytest.fixture(scope="module")
def fmt(tmp_path_factory):
    so = tmp_path_factory.mktemp("format_harness") / "libformat_harness.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", str(ROOT / "tests" / "native" / "format_harness.cpp"),
                    "-I", str(ROOT / "learningorchestra_b200" / "csrc"), "-o", str(so)], check=True)
    lib = C.CDLL(str(so))

    def run(values, status):
        """(lengths int32[n] with -1 for a cell that cannot be formatted, chars uint8, offsets int64[n+1])"""
        bits = np.ascontiguousarray(np.asarray(values, dtype=np.float64)).view(np.uint64)
        st = np.ascontiguousarray(np.broadcast_to(np.asarray(status, dtype=np.uint8), bits.shape))
        n = bits.shape[0]
        lens = np.zeros(n, dtype=np.int32)
        lib.format_lengths(bits.ctypes.data_as(C.c_void_p), st.ctypes.data_as(C.c_void_p), C.c_int64(n),
                           lens.ctypes.data_as(C.c_void_p))
        offsets = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(np.maximum(lens, 0), out=offsets[1:])
        chars = np.zeros(int(offsets[-1]) + 1, dtype=np.uint8)
        written = np.zeros(n, dtype=np.int32)
        lib.format_write(bits.ctypes.data_as(C.c_void_p), st.ctypes.data_as(C.c_void_p), C.c_int64(n),
                         offsets.ctypes.data_as(C.c_void_p), chars.ctypes.data_as(C.c_void_p), written.ctypes.data_as(C.c_void_p))
        assert np.array_equal(written, lens)                 # the two passes agree on every length
        return lens, chars[:-1], offsets
    return run


def bits_to_float(b):
    return struct.unpack("<d", struct.pack("<Q", b & (2 ** 64 - 1)))[0]


def expected(v, s):
    return "" if s == EMPTY else repr(v) if s == FLOAT else str(int(v))


def check(fmt, values, status):
    """Byte for byte against Python, and every text reads back as the same binary64."""
    values = [float(v) for v in values]
    status = list(np.broadcast_to(np.asarray(status, dtype=np.uint8), (len(values),)).tolist())
    lens, chars, offsets = fmt(values, status)
    exp = [expected(v, s) for v, s in zip(values, status)]
    exp_lens = np.fromiter((len(e) for e in exp), dtype=np.int64, count=len(exp))
    raw = chars.tobytes()
    if not (np.array_equal(lens, exp_lens) and raw == "".join(exp).encode()):
        for i, (v, e) in enumerate(zip(values, exp)):
            got = raw[offsets[i]:offsets[i + 1]].decode()
            assert got == e, (i, v.hex(), status[i], got, e)
    assert lens.max(initial=0) <= 310
    assert all(lens[i] <= 24 for i in range(len(values)) if status[i] == FLOAT)
    for v, s, t in zip(values, status, exp):
        if s == EMPTY:
            continue
        back = float(t)
        if math.isnan(v):
            assert math.isnan(back)
        else:
            assert struct.pack("<d", back) == struct.pack("<d", v if s == FLOAT or v != 0 else 0.0), (v, t)
        if s == INTEGER:
            assert int(t) == int(v)


def with_neighbours(vs):
    out = []
    for v in vs:
        out += [v, math.nextafter(v, math.inf), math.nextafter(v, -math.inf)]
    return [x for x in out if math.isfinite(x)]


SPECIAL_BITS = [0x0, 0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000, 0xFFF8000000000000,
                0x7FF0000000000001, 0x7FF8000000000001, 0xFFF0000000000001, 0x7FFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF,
                0x7FF4000000000000, 0xFFF800000000ABCD]
EDGES = [5e-324, bits_to_float(0x000FFFFFFFFFFFFF), 2.2250738585072014e-308, 1.7976931348623157e308,
         1e-4, 1e-5, 1e15, 1e16, 9999999999999998.0, 0.1, 0.2, 0.3, 0.30000000000000004, 1.0, 3.0, 1.5, 1e22, 1e23, 1e300,
         123456789012345680.0, 0.00012345, 1.5e-7, 12345678901234567.0, 1234567890123456.7, 1.7976931348623157e+308 / 3]


def test_specials_and_edges_repr(fmt):
    values = [bits_to_float(b) for b in SPECIAL_BITS]
    values += with_neighbours(EDGES)
    values += with_neighbours([2.0 ** 53, 2.0 ** 63, 2.0 ** 64]) + [2.0 ** 53 + 2, 2.0 ** 53 - 1]
    values += [-v for v in values]
    check(fmt, values, FLOAT)
    lens, chars, _ = fmt([bits_to_float(b) for b in SPECIAL_BITS], FLOAT)
    assert chars.tobytes() == b"0.0-0.0inf-infnannannannannannannannannan"      # every NaN prints "nan"


def test_every_power_of_ten_and_of_two_with_neighbours(fmt):
    tens = [float(f"1e{k}") for k in range(-323, 309)]
    twos = [math.ldexp(1.0, k) for k in range(-1074, 1024)]
    values = with_neighbours(tens) + with_neighbours(twos)
    check(fmt, values + [-v for v in values], FLOAT)


def test_notation_switch_points(fmt):
    """Positional for -4 < decpt <= 16 (integral values get ".0"), exponent form with two or three digits outside."""
    lens, chars, offsets = fmt([1e-4, 1e-5, 1e15, 1e16, 9999999999999998.0, 0.1, 0.3, 5e-324, 1.5e-7, 1e22, -1e100], FLOAT)
    got = [chars.tobytes()[offsets[i]:offsets[i + 1]].decode() for i in range(len(lens))]
    assert got == ["0.0001", "1e-05", "1000000000000000.0", "1e+16", "9999999999999998.0", "0.1", "0.3", "5e-324",
                   "1.5e-07", "1e+22", "-1e+100"]


def test_round_decimals_and_ties(fmt):
    """Values that are short exact decimals: the trailing-zero and exact-bound branches of Ryu."""
    values = [float(k * 10 ** j) for k in range(1, 1000) for j in range(0, 24)]
    values += [k / 10 ** j for k in range(1, 1000) for j in range(1, 24)]
    values += [float(m) * 2.0 ** e for m in (1, 3, 5, 7, 9, 15, 25, 125, 2 ** 52 + 1, 2 ** 53 - 1) for e in range(-60, 80)]
    check(fmt, values, FLOAT)


def test_random_bit_patterns(fmt):
    rng = np.random.default_rng(20261015)
    bits = rng.integers(0, 2 ** 64, size=2_000_000, dtype=np.uint64, endpoint=False)
    values = bits.view(np.float64)
    lens, chars, offsets = fmt(values, FLOAT)
    exp = [repr(v) for v in values.tolist()]
    assert chars.tobytes() == "".join(exp).encode()
    assert lens.tolist() == [len(e) for e in exp]
    # read back, bit for bit (NaN as NaN)
    back = np.array([float(e) for e in exp])
    nan = np.isnan(values)
    assert np.array_equal(np.isnan(back), nan)
    assert np.array_equal(back[~nan].view(np.uint64), values[~nan].view(np.uint64))
    # short-significand doubles (random decimals of up to 17 digits) exercise the shortest-digit search differently
    dec = np.array([float(f"{rng.integers(1, 10 ** 17)}e{rng.integers(-330, 300)}") for _ in range(200_000)])
    check(fmt, dec[np.isfinite(dec) & (dec != 0)], FLOAT)


def test_integer_path_every_exponent(fmt):
    """str(int(v)) of integral doubles from 1 to DBL_MAX: the u64 loop below 2^64, the 1024-bit integer above."""
    rng = np.random.default_rng(7)
    values = [0.0, -0.0, 1.0, -1.0, 1e22, 1e300, 1.7976931348623157e308, -1.7976931348623157e308, 2.0 ** 64 - 2048]
    for e in range(0, 1024):
        values.append(math.ldexp(1.0, e))
        values.append(math.ldexp(float(2 ** 53 - 1), e - 52) if e >= 52 else float(2 ** (e + 1) - 1))
        for _ in range(3):
            m = int(rng.integers(2 ** 52, 2 ** 53))
            v = math.ldexp(float(m), e - 52)
            values.append(float(math.floor(v)) if rng.random() < 0.5 else -float(math.floor(v)))
    values += with_neighbours([2.0 ** 53, 2.0 ** 63, 2.0 ** 64, 1e16, 1e22])
    assert all(math.isfinite(v) and v == math.floor(v) for v in values)
    check(fmt, values, INTEGER)
    lens, _, _ = fmt([1.7976931348623157e308, -1.7976931348623157e308], INTEGER)
    assert lens.tolist() == [309, 310]


def test_cells_that_cannot_be_formatted(fmt):
    lens, _, _ = fmt([1.0, 1.0, 0.5, math.inf, math.nan, 5e-324, 2.0, 7.0, 1.0], [3, 4, 1, 1, 1, 1, 1, 2, 255])
    assert lens.tolist() == [-1, -1, -1, -1, -1, -1, 1, 0, -1]


# ---- DataType routing ---------------------------------------------------------------------------------------------
class FormatEngine(OracleEngine):
    """The oracle stand-in plus a formatter that is Python's own repr / str(int); it records what it was given so the
    tests see which cells the executor sends to the device and with which status."""

    def __init__(self, fail=False):
        self.calls, self.fail = [], fail

    def format_number_host(self, values, status):
        values, status = np.asarray(values, dtype=np.float64), np.asarray(status, dtype=np.uint8)
        self.calls.append((values.copy(), status.copy()))
        if self.fail:
            raise RuntimeError("device formatter failed")
        texts = [expected(v, s).encode() for v, s in zip(values.tolist(), status.tolist())]
        offsets = np.zeros(len(texts) + 1, dtype=np.int64)
        np.cumsum([len(t) for t in texts], out=offsets[1:])
        return np.frombuffer(b"".join(texts), dtype=np.uint8).copy(), offsets


def _load(name):
    return json.loads((GOLD / name).read_text())


def test_columnar_number_column_goes_to_the_formatter_in_one_call():
    values = np.array([1.5, 3.0, np.nan, -0.0, 1e22, np.inf, 0.1, 7.0, np.nan], dtype=np.float64)
    valid = np.array([1, 1, 0, 1, 1, 1, 1, 1, 1], dtype=bool)
    is_int = np.array([0, 1, 0, 1, 1, 0, 0, 1, 0], dtype=bool)
    col = NumberColumn(values, valid, is_int)
    host = ["" if v is None else str(v) for v in col.to_pylist()]         # what the reference's str() makes of the cells
    db = ColumnarDatabase()
    db.ingest_columns("t", {"x": col})
    eng = FormatEngine()
    job = DataType(db, utils.DataTypeMetadata(db), engine=eng)
    job.convert_existent_file("t", {"x": "string"})
    job.wait(60)
    assert db.find_one("t", {"_id": 0})["finished"] is True
    assert len(eng.calls) == 1
    assert eng.calls[0][1].tolist() == [FLOAT, INTEGER, EMPTY, INTEGER, INTEGER, FLOAT, FLOAT, INTEGER, FLOAT]
    new = db.column("t", "x")
    import pyarrow as pa
    assert isinstance(new, TextColumn) and new.arr.type == pa.large_string() and new.arr.null_count == 0
    assert new.to_pylist() == host == ["1.5", "3", "", "0", "10000000000000000000000", "inf", "0.1", "7", "nan"]


def test_documents_send_only_binary64_numbers_to_the_formatter():
    cells = [None, 1.5, 3, True, False, 2 ** 60 + 1, 2 ** 53, 10 ** 400, -(10 ** 22), "abc", "", [1, 2], -0.0,
             float("nan"), 1e22, {"a": 1}, 0]
    db = utils.Database()
    db.insert_one_in_file("t", rsem.dataset_metadata("t", ["v"]))
    db.insert_many_in_file("t", [{"_id": i + 1, "v": c} for i, c in enumerate(cells)])
    eng = FormatEngine()
    job = DataType(db, utils.DataTypeMetadata(db), engine=eng)
    job.convert_existent_file("t", {"v": "string"})
    job.wait(60)
    assert db.find_one("t", {"_id": 0})["finished"] is True
    got = [d["v"] for d in db.find("t", {}) if d["_id"] != 0]
    assert got == ["" if c is None else str(c) for c in cells]
    assert len(eng.calls) == 1
    values, status = eng.calls[0]
    sent = [1.5, 3, 2 ** 53, -(10 ** 22), -0.0, float("nan"), 1e22, 0]     # floats, and ints that are exactly a double
    assert status.tolist() == [FLOAT, INTEGER, INTEGER, INTEGER, FLOAT, FLOAT, FLOAT, INTEGER]
    assert all((math.isnan(a) and math.isnan(b)) or a == b for a, b in zip(values.tolist(), sent))


def _string_cast(db, name, fields, eng):
    job = DataType(db, utils.DataTypeMetadata(db), engine=eng)
    job.convert_existent_file(name, {f: "string" for f in fields})
    job.wait(60)
    assert db.find_one(name, {"_id": 0})["finished"] is True
    return sorted([d["_id"]] + [d[f] for f in fields] for d in db.find(name, {}) if d["_id"] != 0)


def test_titanic_string_cast_equals_the_reference_on_both_stores(tmp_path):
    gold_n, gold_s = _load("reference_datatype_number.json"), _load("reference_datatype_string.json")
    # documents: the reference's own "number" result, then "string"
    db = utils.Database()
    db.insert_one_in_file("t", rsem.dataset_metadata("t", gold_n["fields"]))
    db.insert_many_in_file("t", [dict(zip(["_id"] + gold_n["fields"], row)) for row in gold_n["rows"]])
    eng = FormatEngine()
    assert _string_cast(db, "t", gold_s["fields"], eng) == gold_s["rows"]
    assert len(eng.calls) == len(gold_s["fields"])
    # columns: CSV ingest, "number", then "string" -- every number column in one formatter call
    g = _load("titanic_shaped_input.json")
    path = tmp_path / "titanic.csv"
    import csv
    with path.open("w", newline="") as f:
        csv.writer(f, lineterminator="\n").writerows([g["headers"]] + g["rows"])
    db = ColumnarDatabase()
    db.ingest_csv("titanic", str(path))
    eng = FormatEngine()
    job = DataType(db, utils.DataTypeMetadata(db), engine=eng)
    job.convert_existent_file("titanic", {f: "number" for f in gold_n["fields"]})
    job.wait(60)
    assert all(isinstance(db.column("titanic", f), NumberColumn) for f in gold_s["fields"])
    assert _string_cast(db, "titanic", gold_s["fields"], eng) == gold_s["rows"]
    assert len(eng.calls) == len(gold_s["fields"])
    assert all(isinstance(db.column("titanic", f), TextColumn) for f in gold_s["fields"])


def test_a_failing_formatter_fails_the_job_without_a_host_retry():
    for db in (utils.Database(), ColumnarDatabase()):
        db.insert_one_in_file("t", rsem.dataset_metadata("t", ["v"]))
        db.insert_many_in_file("t", [{"_id": 1, "v": 1.5}, {"_id": 2, "v": 2}])
        job = DataType(db, utils.DataTypeMetadata(db), engine=FormatEngine(fail=True))
        job.convert_existent_file("t", {"v": "string"})
        with pytest.raises(RuntimeError, match="device formatter failed"):
            job.wait(60)
        meta = db.find_one("t", {"_id": 0})
        assert meta["finished"] is False and "device formatter failed" in meta["exception"]
        assert [d["v"] for d in db.find("t", {}) if d["_id"] != 0] == [1.5, 2]          # untouched
