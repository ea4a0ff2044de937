"""CPU: the streaming reader's window bookkeeping (csv::StreamWindow, csv::segment_last_end, absolute records and
positions) compiled with g++ (tests/native/csv_stream_harness.cpp) and run on bodies pushed in pieces through small
windows, against the reference's own csv.reader call (csv_oracle.csv_reference_rows) and the single-shot reader's
decomposition (tests/native/csv_harness.cpp); the lo_csv_window layout."""
import ctypes as C
import random
import subprocess

import numpy as np
import pytest

from csv_oracle import csv_reference_rows
from test_csv_cpu import BUILD, CSRC, HAND, ROOT, harness, random_cuts, to_rows  # noqa: F401  (harness: a fixture)


@pytest.fixture(scope="module")
def stream_harness():
    src, hdr, so = ROOT / "tests" / "native" / "csv_stream_harness.cpp", CSRC / "csv_reader.cuh", BUILD / "libcsv_stream_harness.so"
    if not so.exists() or so.stat().st_mtime < max(src.stat().st_mtime, hdr.stat().st_mtime):
        BUILD.mkdir(exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-fPIC", "-shared", str(src), "-I", str(CSRC), "-o", str(so)],
                       check=True)
    lib = C.CDLL(str(so))
    lib.csv_stream_read.restype = C.c_int64
    return lib


def stream_info(lib, body: bytes, pieces, window: int, seg: int):
    """(info int64[6], offsets, chars) of the body pushed in pieces (cut positions from 0 to len(body))."""
    n = len(body)
    pieces = np.asarray(pieces, dtype=np.int64)
    buf = np.frombuffer(body + b"\0", dtype=np.uint8)
    info = np.zeros(6, np.int64)
    offsets = np.zeros(2 * n + 4, np.int64)
    chars = np.zeros(n + 1, np.uint8)
    rc = lib.csv_stream_read(buf.ctypes.data_as(C.c_void_p), pieces.ctypes.data_as(C.c_void_p), C.c_int64(len(pieces) - 1),
                             C.c_int64(window), C.c_int64(seg), info.ctypes.data_as(C.c_void_p),
                             offsets.ctypes.data_as(C.c_void_p), C.c_int64(offsets.size), chars.ctypes.data_as(C.c_void_p),
                             C.c_int64(chars.size))
    assert rc >= 0
    return info, offsets, chars


def single_info(lib, body: bytes):
    n = len(body)
    bounds = np.asarray([0, n], dtype=np.int64)
    buf = np.frombuffer(body + b"\0", dtype=np.uint8)
    info = np.zeros(6, np.int64)
    offsets = np.zeros(2 * n + 4, np.int64)
    chars = np.zeros(n + 1, np.uint8)
    assert lib.csv_read(buf.ctypes.data_as(C.c_void_p), C.c_int64(n), bounds.ctypes.data_as(C.c_void_p), C.c_int64(1),
                        info.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), C.c_int64(offsets.size),
                        chars.ctypes.data_as(C.c_void_p)) == 0
    return info


def check(stream_lib, single_lib, body, pieces, window, seg, exp=None):
    info, offsets, chars = stream_info(stream_lib, body, pieces, window, seg)
    got = to_rows(info[0], info[1], chars[:info[2]].tobytes(), offsets, info[3], info[4])
    assert got == (exp if exp is not None else csv_reference_rows(body)), (body, pieces, window, seg)
    assert list(info) == list(single_info(single_lib, body)), (body, pieces, window, seg)


def even(n, size):
    return list(range(0, n, size)) + [n] if n else [0, 0]


@pytest.mark.parametrize("body", HAND, ids=range(len(HAND)))
def test_hand_cases_every_piece_and_window(stream_harness, harness, body):
    exp = csv_reference_rows(body)
    rng = random.Random(len(body) * 7 + 1)
    for window in (16, 64, 256, max(len(body), 1)):
        for seg in (3, 256):
            for size in (1, 2, 3, 7):
                check(stream_harness, harness, body, even(len(body), size), window, seg, exp)
            for _ in range(3):
                check(stream_harness, harness, body, random_cuts(rng, len(body)) if body else [0, 0], window, seg, exp)


@pytest.mark.parametrize("window", [1, 2, 5])
def test_windows_smaller_than_a_record_grow(stream_harness, harness, window):
    """No record ends in the window: it doubles until one does; the result does not change."""
    body = b'h1,h2\n"a long\r\nquoted field",x\r\n\n' + b"plain,row\n" * 3 + "é€😀,\"\"\"\"\n".encode()
    for size in (1, 3, len(body)):
        check(stream_harness, harness, body, even(len(body), size), window, 2)


def test_breaks_and_sequences_straddling_the_cut(stream_harness, harness):
    """A run of breaks, a UTF-8 sequence or a "" pair split between windows and between pieces."""
    heads = [b"a,b\n", b"a,b\r", b"a,b\r\n"]
    tails = [b"\n1,2\n", b"\r\n1,2\r\n", "é,€\n😀,x\n".encode(), b'"x""y",2\n', b'"q\r\n\r\nr",2']
    for h in heads:
        for t in tails:
            body = h + t + b"3,4"
            for window in range(1, len(body) + 2):
                for cut in range(len(body) + 1):
                    check(stream_harness, harness, body, [0, cut, len(body)] if cut else [0, len(body)], window, 4)


def test_random_bodies(stream_harness, harness):
    """100 000 bodies over {, " \\r \\n a space é-bytes NUL 0xff}, in random pieces through random small windows."""
    rng = random.Random(20261017)
    alphabet = [b",", b"\"", b"\r", b"\n", b"a", b" ", "é".encode(), b"\xc3", b"\xa9", b"\x00", b"\xff"]
    weights = [6, 6, 3, 4, 6, 2, 2, 1, 1, 0.3, 0.3]
    for _ in range(100_000):
        body = b"".join(rng.choices(alphabet, weights, k=rng.randint(0, 30)))
        pieces = random_cuts(rng, len(body)) if body else [0, 0]
        check(stream_harness, harness, body, pieces, rng.choice((1, 2, 3, 4, 8, 16, 64)), rng.choice((1, 2, 3, 5, 256)))


def test_csv_window_layout():
    """lo_csv_window as the C compiler lays it out == the ctypes mirror."""
    from learningorchestra_b200 import _native as N
    src = BUILD / "csv_window_layout.c"
    exe = BUILD / "csv_window_layout"
    BUILD.mkdir(exist_ok=True)
    fields = ("consumed", "records", "first_record", "ncols", "chars", "peak_device_bytes", "done", "pad")
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "loexec.h"\nint main(void) {\n'
                   '  printf("%zu %lld", sizeof(lo_csv_window), (long long)LO_CSV_STREAM_WINDOW);\n'
                   + "".join(f'  printf(" %zu", offsetof(lo_csv_window, {f}));\n' for f in fields)
                   + '  printf("\\n");\n  return 0;\n}\n')
    subprocess.run(["gcc", "-std=c11", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    W = N.CsvWindow
    assert [int(x) for x in out] == [C.sizeof(W), N.LO_CSV_STREAM_WINDOW] + [getattr(W, f).offset for f in fields]
