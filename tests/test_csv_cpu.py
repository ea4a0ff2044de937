"""CPU: the upload reader's rules (csrc/csv_reader.cuh, __host__ __device__) compiled with g++ and run through the
device reader's segment decomposition (tests/native/csv_harness.cpp), against the reference's own csv.reader call
(csv_oracle.csv_reference_rows); the oracle itself against the reference's behaviour; the lo_csv_info layout."""
import codecs
import ctypes as C
import random
import subprocess
from pathlib import Path

import numpy as np
import pytest

from csv_oracle import KINDS, csv_reference_rows

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "learningorchestra_b200" / "csrc"
BUILD = ROOT / "tests" / "native" / "_build"


@pytest.fixture(scope="module")
def harness():
    src, hdr, so = ROOT / "tests" / "native" / "csv_harness.cpp", CSRC / "csv_reader.cuh", BUILD / "libcsv_harness.so"
    if not so.exists() or so.stat().st_mtime < max(src.stat().st_mtime, hdr.stat().st_mtime):
        BUILD.mkdir(exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-fPIC", "-shared", str(src), "-I", str(CSRC), "-o", str(so)],
                       check=True)
    lib = C.CDLL(str(so))
    lib.csv_read.restype = C.c_int
    return lib


def read(lib, body: bytes, bounds=None):
    """(header, rows, failure) through the harness, in the oracle's form; bounds: segment cuts (default: one)."""
    n = len(body)
    bounds = np.asarray(bounds if bounds is not None else [0, n], dtype=np.int64)
    buf = np.frombuffer(body + b"\0", dtype=np.uint8)
    info = np.zeros(6, np.int64)
    offsets = np.zeros(2 * n + 4, np.int64)
    chars = np.zeros(n + 1, np.uint8)
    rc = lib.csv_read(buf.ctypes.data_as(C.c_void_p), C.c_int64(n), bounds.ctypes.data_as(C.c_void_p),
                      C.c_int64(len(bounds) - 1), info.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p),
                      C.c_int64(offsets.size), chars.ctypes.data_as(C.c_void_p))
    assert rc == 0
    return to_rows(info[0], info[1], chars[:info[2]].tobytes(), offsets, info[3], info[4])


def to_rows(records, ncols, chars, offsets, fail_record, fail_kind):
    """The reader's columns back to the oracle's (header, rows, failure)."""
    off = np.asarray(offsets[:ncols * (records + 1)]).reshape(ncols, records + 1) if records else None
    cell = lambda c, r: chars[off[c, r]:off[c, r + 1]].decode("utf-8")
    header = [cell(c, 0) for c in range(ncols)] if records else None
    rows = [[cell(c, r) for c in range(ncols)] for r in range(1, records)]
    failure = None if fail_kind == 0 else (KINDS[fail_kind], int(fail_record))
    return header, rows, failure


def random_cuts(rng, n):
    cuts, p = [0], 0
    while p < n:
        p = min(n, p + rng.choice((1, 1, 2, 3, 5, 8, 64, 256)))
        cuts.append(p)
    return cuts


HAND = [
    # rule 1: lines
    b"a,b\n1,2", b"a,b\r\n1,2\r\n", b"a,b\r\r1,2\n\n\n", b"\n\na,b\n\n1,2\n", b"a,b\n\"x\ny\",2", b"a,b\n\"x\r\n\r\ny\",2\n",
    b"a,b\r1,2\r", b"", b"\n\r\n", b"a\n",
    # rule 2: fields
    b"a,b\na\"b,c", b"a,b\n\"a\"\"b\",c", b"a,b\n\"ab\"cd,e", b"a,b\n \"x,y\",2", b"a,b\n\"x,y\" ,2", b"a,b\n\"unterminated,2",
    b"a,b\n1,\"", b"a,b\n,\n\"\",\"\"", b"a,b\n\"\"\"\",x", b"a,b\n\"a\"\"\n\"\"b\",c", b"\"h\"\"1\",h2\n1,2", b"a,b\n1,2,3",
    b"a,b\n1,2,\"3\n4\"\n5,6",
    # rule 6: rows
    b"a,b\n1", b"a,b\n1,2\n3\n4,5", b"a,b,c\n,,\n", b"a\n\"\"",
    # rule 4: UTF-8
    "﻿id,name\n1,é\n".encode(), "h\nö€😀\n".encode(), b"h\n\xc0\x80\n", b"h\n\xe0\x80\x80\n", b"h\n\xed\xa0\x80\n",
    b"h\n\xf5\x80\x80\x80\n", b"h\n\xf4\x90\x80\x80\n", b"h\n\xff\n", b"h\n\x80\n", b"h\nok\n\xc3a\n", b"h\n\xc3\n2\n",
    b"h\n\xe2\x82\n", b"h\n1\n\xe2\x82", b"h\n\"\xc3\n\xa9\"\n", b"h\n\xc3\xa9\xa9\n", b"h\n\xf0\x9f\x98\n", b"\xff\n1\n",
    # rule 5: NUL
    b"h\n1\n\x002\n", b"h\n\"a\nb\x00\"\n", b"h\x00\n1\n", b"h,i\n1,\x00\n",
]


def test_oracle_matches_the_issue_table():
    assert csv_reference_rows(b"a,b\n\"x\ny\",2") == (["a", "b"], [["xy", "2"]], None)
    assert csv_reference_rows(b"a,b\n1,2,3") == (["a", "b"], [["1", "2"]], None)
    assert csv_reference_rows(b"a,b\n \"x,y\",2") == (["a", "b"], [[' "x', 'y"']], None)
    assert csv_reference_rows(b"a,b\n0,0\n1") == (["a", "b"], [["0", "0"]], ("short_row", 2))
    assert csv_reference_rows(b"") == (None, [], ("empty", 0))
    assert csv_reference_rows(b"a,b\n\"ab\"cd,a\"b") == (["a", "b"], [["abcd", 'a"b']], None)
    assert csv_reference_rows(b"a,b\n\"a\"\"b\",\"open") == (["a", "b"], [['a"b', "open"]], None)


def test_oracle_runs_the_stdlib_reader_where_the_rules_agree():
    """On NUL-free bodies whose lines are whole UTF-8, the oracle is csv.reader(codecs.iterdecode(...)) verbatim."""
    import csv
    rng = random.Random(7)
    for _ in range(3000):
        body = b"".join(rng.choice([b",", b"\"", b"\r", b"\n", b"a", b" ", "é".encode()]) for _ in range(rng.randint(0, 24)))
        header, rows, failure = csv_reference_rows(body)
        recs = list(csv.reader(codecs.iterdecode(body.splitlines(), "utf-8"), delimiter=",", quotechar='"'))
        if not recs:
            assert failure == ("empty", 0)
            continue
        assert header == recs[0]
        short = [i for i, r in enumerate(recs[1:], 1) if len(r) < len(recs[0])]
        stop = short[0] if short else len(recs)
        assert rows == [r[:len(recs[0])] for r in recs[1:stop]]
        assert failure == (("short_row", short[0]) if short else None)


def test_oracle_failures():
    assert csv_reference_rows(b"h\n1\n\x002\n") == (["h"], [["1"]], ("nul", 2))
    assert csv_reference_rows(b"h\x00\n1\n") == (None, [], ("nul", 0))
    assert csv_reference_rows(b"h\n1\n\xff\n") == (["h"], [["1"]], ("bad_utf8", 2))
    assert csv_reference_rows(b"h\n1\n\xc3\n\xa9\n") == (["h"], [["1"]], ("unsupported", 2))
    ok = ("h\n" + "é" * 131072 + "\n").encode()
    assert csv_reference_rows(ok) == (["h"], [["é" * 131072]], None)
    assert csv_reference_rows(b"h\n1\n" + b"a" * 131073 + b"\n") == (["h"], [["1"]], ("field_limit", 2))
    # the field limit before a NUL on the same line wins; a NUL before the limit wins
    assert csv_reference_rows(b"h\n" + b"a" * 131073 + b"\x00\n")[2] == ("field_limit", 1)
    assert csv_reference_rows(b"h\n\x00" + b"a" * 131073 + b"\n")[2] == ("nul", 1)


@pytest.mark.parametrize("body", HAND, ids=range(len(HAND)))
def test_hand_cases_every_decomposition(harness, body):
    exp = csv_reference_rows(body)
    assert read(harness, body) == exp
    for size in (1, 2, 3, 7):
        assert read(harness, body, list(range(0, len(body), size)) + [len(body)] if body else [0, 0]) == exp, size
    rng = random.Random(len(body))
    for _ in range(5):
        assert read(harness, body, random_cuts(rng, len(body))) == exp


@pytest.mark.parametrize("cp,n,fails", [("a", 131072, False), ("a", 131073, True), ("é", 131072, False),
                                         ("é", 131073, True), ("€", 131073, True), ("😀", 131072, False)])
def test_field_limit_in_code_points(harness, cp, n, fails):
    for body in (("h\n1\n" + cp * n + "\n2\n").encode(), ("h\n1\n\"" + cp * (n - 1) + '""' + "\"\n2\n").encode(),
                 ("h\n1\n\"" + cp * (n // 2) + "\n\n" + cp * (n - n // 2) + "\"\n2\n").encode()):
        exp = csv_reference_rows(body)
        assert (exp[2] == ("field_limit", 2)) == fails
        rng = random.Random(n)
        assert read(harness, body, random_cuts(rng, len(body))) == exp


@pytest.mark.parametrize("seq", [b"\xc0\xaf", b"\xc1\xbf", b"\xe0\x80\xaf", b"\xe0\x9f\xbf", b"\xed\xa0\x80", b"\xed\xbf\xbf",
                                 b"\xf0\x80\x80\xaf", b"\xf0\x8f\xbf\xbf", b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xfe",
                                 b"\xff", b"\x80", b"\xbf", b"\xc3\xa9\xa9", b"\xe2\x82", b"\xe2\x82a", b"\xf0\x9f\x98",
                                 b"\xc3", b"\xe2\x82\xac", b"\xf4\x8f\xbf\xbf", b"\xed\x9f\xbf"])
def test_utf8_classes_against_the_decoder(harness, seq):
    for body in (b"h\n1\n" + seq + b"\n2\n", b"h\n1\n\"" + seq + b"\"\n2\n", b"h\n1\n" + seq, b"h\n1\n" + seq + b"x\n"):
        exp = csv_reference_rows(body)
        if exp[2] is None:
            seq.decode("utf-8")          # accepted only when the decoder accepts the line
        assert read(harness, body) == exp
        assert read(harness, body, list(range(len(body) + 1))) == exp


def test_random_bodies(harness):
    """100 000 bodies over {, " \\r \\n a space é-bytes NUL 0xff}, each cut into random segments."""
    rng = random.Random(20261016)
    alphabet = [b",", b"\"", b"\r", b"\n", b"a", b" ", "é".encode(), b"\xc3", b"\xa9", b"\x00", b"\xff"]
    weights = [6, 6, 3, 4, 6, 2, 2, 1, 1, 0.3, 0.3]
    bad = 0
    for i in range(100_000):
        body = b"".join(rng.choices(alphabet, weights, k=rng.randint(0, 30)))
        exp = csv_reference_rows(body)
        got = read(harness, body, random_cuts(rng, len(body)) if body else [0, 0])
        if got != exp:
            bad += 1
            assert got == exp, body
    assert bad == 0


def test_csv_info_layout():
    """lo_csv_info as the C compiler lays it out == the ctypes mirror."""
    from learningorchestra_b200 import _native as N
    src = BUILD / "csv_info_layout.c"
    exe = BUILD / "csv_info_layout"
    BUILD.mkdir(exist_ok=True)
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "loexec.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(lo_csv_info), offsetof(lo_csv_info, records),\n'
                   '         offsetof(lo_csv_info, ncols), offsetof(lo_csv_info, chars), offsetof(lo_csv_info, fail_record),\n'
                   '         offsetof(lo_csv_info, fail_kind), offsetof(lo_csv_info, fail_pos));\n'
                   '  printf("%d %d %d %d %d %d %d\\n", LO_CSV_OK, LO_CSV_SHORT_ROW, LO_CSV_FIELD_LIMIT, LO_CSV_BAD_UTF8,\n'
                   '         LO_CSV_NUL, LO_CSV_UNSUPPORTED, LO_CSV_EMPTY);\n  return 0;\n}\n')
    subprocess.run(["gcc", "-std=c11", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    I = N.CsvInfo
    assert [int(x) for x in out[0].split()] == [C.sizeof(I), I.records.offset, I.ncols.offset, I.chars.offset,
                                                I.fail_record.offset, I.fail_kind.offset, I.fail_pos.offset]
    assert [int(x) for x in out[1].split()] == [N.LO_CSV_OK, N.LO_CSV_SHORT_ROW, N.LO_CSV_FIELD_LIMIT, N.LO_CSV_BAD_UTF8,
                                                N.LO_CSV_NUL, N.LO_CSV_UNSUPPORTED, N.LO_CSV_EMPTY]
    assert [KINDS.index(k) for k in ("ok", "short_row", "field_limit", "bad_utf8", "nul", "unsupported", "empty")] == \
        list(range(7))
