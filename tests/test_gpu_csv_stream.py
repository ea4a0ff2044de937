"""GPU: the streaming CSV reader (lo_csv_stream_*, Engine.read_csv_stream) against the reference's own csv.reader call
(csv_oracle.csv_reference_rows) and the single-shot reader (lo_csv_read_host) on the same body: pieces cut anywhere,
windows as small as a byte, failures after several windows, and device memory bounded by the window on a 4 GiB body."""
import ctypes as C
import io
import random

import numpy as np
import pytest

from csv_oracle import KINDS, csv_reference_rows
from learningorchestra_b200 import _native as N
from test_csv_cpu import HAND, random_cuts
from test_gpu_csv import device_rows

pytestmark = pytest.mark.gpu
P = C.c_void_p


def pushed_rows(engine, body: bytes, cuts, window: int, last_with_data: bool = False):
    """(header, rows, failure (kind, record, pos), peak device bytes) of the body pushed through the C API in the
    pieces cuts[i]..cuts[i+1], then a zero-byte last push (or last = 1 on the final piece)."""
    lib, ctx = engine._lib, engine._ctx
    buf = np.frombuffer(body + b"\0", np.uint8)
    st, win, info, t = P(), N.CsvWindow(), N.CsvInfo(), N.HostTiming()
    N.check(lib.lo_csv_stream_open(ctx, window, C.byref(st)))
    header, cols = None, []
    pieces = [(cuts[i], cuts[i + 1], last_with_data and i == len(cuts) - 2) for i in range(len(cuts) - 1)]
    if not last_with_data or not pieces:
        pieces.append((len(body), len(body), True))
    try:
        for a, b, last in pieces:
            off = a
            while True:
                N.check(lib.lo_csv_stream_push(st, P(buf.ctypes.data + off), b - off, int(last), C.byref(win),
                                               C.byref(info), C.byref(t)))
                assert 0 <= win.consumed <= b - off
                if win.records:
                    k, nc = win.records, win.ncols
                    offsets = np.zeros((nc, k + 1), np.int64)
                    chars = np.zeros(max(win.chars, 1), np.uint8)
                    N.check(lib.lo_csv_stream_columns(st, offsets.ctypes.data_as(P), chars.ctypes.data_as(P), chars.size,
                                                      C.byref(t)))
                    raw = chars.tobytes()
                    cells = [[raw[offsets[c, r]:offsets[c, r + 1]].decode("utf-8") for c in range(nc)] for r in range(k)]
                    if win.first_record == 0:
                        header, cells = cells[0], cells[1:]
                    cols.extend(cells)
                off += win.consumed
                if win.done or (off >= b and not last):
                    break
            if win.done:
                break
        assert win.done
    finally:
        N.check(lib.lo_csv_stream_free(st))
    assert info.records == (len(cols) + 1 if header is not None else 0)
    failure = None if info.fail_kind == N.LO_CSV_OK else (int(info.fail_kind), int(info.fail_record), int(info.fail_pos))
    return header, cols, failure, int(win.peak_device_bytes)


def single(engine, body: bytes):
    """(header, rows, failure (kind, record, pos)) of lo_csv_read_host."""
    header, nrows, chars, offsets, failure = engine.read_csv_host(body)
    raw = chars.tobytes()
    rows = [[raw[offsets[c, r]:offsets[c, r + 1]].decode("utf-8") for c in range(offsets.shape[0])] for r in range(1, nrows + 1)]
    return header, rows, failure


def oracle_form(failure):
    return None if failure is None else (KINDS[failure[0]], failure[1])


def check(engine, body, cuts, window, exp=None, ref=None, last_with_data=False):
    exp = exp if exp is not None else csv_reference_rows(body)
    ref = ref if ref is not None else single(engine, body)
    header, rows, failure, _ = pushed_rows(engine, body, cuts, window, last_with_data)
    assert (header, rows, oracle_form(failure)) == exp, (body[:200], cuts[:20], window)
    assert (header, rows, failure) == ref, (body[:200], cuts[:20], window)


def even(n, size):
    return list(range(0, n, size)) + [n] if n else [0, 0]


def test_hand_cases(engine):
    rng = random.Random(3)
    for body in HAND:
        exp, ref = csv_reference_rows(body), single(engine, body)
        for window in (1, 5, 64):
            check(engine, body, random_cuts(rng, len(body)) if body else [0, 0], window, exp, ref)
            check(engine, body, even(len(body), 1), window, exp, ref, last_with_data=True)


def test_random_bodies(engine):
    rng = random.Random(20261017)
    alphabet = [b",", b"\"", b"\r", b"\n", b"a", b" ", "é".encode(), b"\xc3", b"\xa9", b"\x00", b"\xff"]
    weights = [6, 6, 3, 4, 6, 2, 2, 1, 1, 0.3, 0.3]
    for _ in range(3000):
        body = b"".join(rng.choices(alphabet, weights, k=rng.randint(0, 40)))
        check(engine, body, random_cuts(rng, len(body)) if body else [0, 0], rng.choice((1, 3, 8, 64)))


def test_bodies_straddling_pieces_and_windows(engine):
    # "\r" and "\n" split between pushes, at every position, through windows around the split
    for body in (b"a,b\r\n1,2\r\n3,4\r\n", b"a,b\r\r\n\n1,2\n\r5,6"):
        for cut in range(1, len(body)):
            for window in (4, 5, 8, 9):
                check(engine, body, [0, cut, len(body)], window)
    # every UTF-8 sequence length split at each byte, and "" split between its quotes
    for cell in ("é", "€", "😀", '"x""y"', '""""'):
        body = ("h,i\n1," + cell + "\n" + cell + ",2\n").encode()
        for cut in range(1, len(body)):
            for window in (6, 7, len(body)):
                check(engine, body, [0, cut, len(body)], window)
    # a quoted multi-line field across more than 10 windows of 64 bytes
    field = "".join(f"line {i}, \"\"q\"\" é\r\n" for i in range(60))
    body = ('a,b\n1,"' + field.replace('""', '""') + '"\n2,3\n').encode()
    assert len(body) > 10 * 64
    check(engine, body, random_cuts(random.Random(1), len(body)), 64)
    # a record many times longer than the starting window: the window grows
    body = b"h1,h2\n" + b"x" * 5000 + b",y\nz,w\n"
    check(engine, body, even(len(body), 333), 64)
    # the 100 KB quoted field of the single-shot boundary test, through 4 KiB windows
    big = b'h,i\n1,"' + ("é,\"\"\n" * 20000).encode() + b'"\n2,3\n'
    check(engine, big, even(len(big), 1000), 4096)


def test_failure_kinds_after_several_windows(engine):
    good = b"a,b\n" + b"".join(b"%d,%d\n" % (i, i * i) for i in range(300))
    cases = {
        N.LO_CSV_SHORT_ROW: b"5\n6,7\n",
        N.LO_CSV_FIELD_LIMIT: b"x" * 131073 + b",5\n",
        N.LO_CSV_BAD_UTF8: b"3,\xff\n5,6\n",
        N.LO_CSV_NUL: b"3,4\x00\n5,6\n",
        N.LO_CSV_UNSUPPORTED: b"\xc3\n\xa9,5\n",
    }
    for kind, bad in cases.items():
        body = good + bad
        ref = single(engine, body)
        assert ref[2][:2] == (kind, 301) and len(ref[1]) == 300
        for window in (64, 1000):
            check(engine, body, even(len(body), 777), window, ref=ref)
            header, rows, failure, _ = pushed_rows(engine, body, [0, len(body)], window)
            assert failure == ref[2] and rows == ref[1]


def test_edges(engine):
    for body in (b"", b"\n\r\n", b"a,b\n", b"a,b", b"a\x00,b\n1,2\n", b"a,b\n1,2", b"a,b\n1,2\n\n\n"):
        for window in (1, 2, 64):
            check(engine, body, even(len(body), 1), window)
            check(engine, body, [0, len(body)] if body else [0, 0], window, last_with_data=True)


def test_read_csv_stream_sources(engine, tmp_path):
    """A path, a binary file object, a text file object and an iterable of bytes: the same columns as read_csv_host."""
    body = ('id,"na,me",text\r\n' + "".join(f'{i},"n""{i}",é{"x" * (i % 50)}\r\n' for i in range(2000))).encode()
    path = tmp_path / "b.csv"
    path.write_bytes(body)
    ref = device_rows(engine, body)
    rng = random.Random(9)
    chunks = [body[a:b] for a, b in zip(*(lambda c: (c[:-1], c[1:]))(random_cuts(rng, len(body))))]
    sources = (lambda: str(path), lambda: path, lambda: io.BytesIO(body), lambda: io.StringIO(body.decode()),
               lambda: iter(chunks))
    for make in sources:
        for window in (1000, None):
            timing = {}
            header, nrows, columns, failure = engine.read_csv_stream(make(), window, timing)
            for col in columns:
                col.validate(full=True)
            rows = [list(r) for r in zip(*(col.to_pylist() for col in columns))]
            assert (header, rows, oracle_form(failure)) == ref
            assert timing["peak_device_bytes"] > 0 and timing["windows"] >= 1


def _block_file(path, reps):
    block = 'id,"quoted, text","multi\r\nline ""é"""\n'.encode()
    with open(path, "wb") as f:
        f.write(b"a,b,c\n")
        chunk = block * (1 << 16)
        for _ in range(reps >> 16):
            f.write(chunk)
        f.write(block * (reps & 0xFFFF))
    return block


def test_bounded_memory_on_a_4_gib_body(engine, tmp_path):
    """A repeated block streamed from a file through a 64 MiB window: the columns by construction, the peak device
    bytes within the bound of include/loexec.h and the same as for a 1 GiB body of the same block."""
    W = 64 << 20
    peaks = {}
    for gib in (1, 4):
        path = tmp_path / f"b{gib}.csv"
        block = _block_file(path, 0)
        reps = (gib << 30) // len(block) + 1
        _block_file(path, reps)
        timing = {}
        header, nrows, columns, failure = engine.read_csv_stream(str(path), W, timing)
        path.unlink()
        assert header == ["a", "b", "c"] and nrows == reps and failure is None
        for col, cell in zip(columns, (b"id", b"quoted, text", b'multiline "\xc3\xa9"')):
            offs = np.frombuffer(col.buffers()[1], np.int64, count=nrows + 1, offset=col.offset * 8)
            assert (np.diff(offs) == len(cell)).all() and offs[0] == 0
            for r in (0, nrows // 2, nrows - 1):
                assert col[r].as_py().encode() == cell
        del columns
        cells = 3 * (W // len(block) + 1)
        bound = 2 * W + (W // 256 + 1) * (8 + 2 * 56) + 64 + 8 * (cells + 3 + 1) + W + (4 << 20)   # + CUB storage
        assert 2 * W < timing["peak_device_bytes"] <= bound, timing
        peaks[gib] = timing["peak_device_bytes"]
    assert peaks[1] == peaks[4]
