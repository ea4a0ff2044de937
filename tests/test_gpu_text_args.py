"""GPU: the four entry points that take a packed text column from the host — ``lo_value_counts_str_host``,
``lo_parse_number_host``, ``lo_parse_number_to_table`` and ``lo_text_upload`` — on one table of malformed arguments and
on one sliced Arrow column with nulls.

Pins what each one refuses (a refusal launches nothing), what each one lets through on purpose (the table parse leaves
backwards offsets to its kernel, which reports the cell as unsupported; only the host group-by insists on
offsets[0] == 0), and what each one copies to the device: the chars span, the n + 1 offsets and the bytes of validity
that cover the column.  Expected values come from ``float()`` and ``collections.Counter``."""
import ctypes as C
from collections import Counter

import numpy as np
import pytest

from learningorchestra_b200 import _native as N
from learningorchestra_b200.columnar import text_buffers

pytestmark = pytest.mark.gpu

ENTRIES = ("value_counts_str", "parse_number", "parse_number_to_table", "text_upload")
TABLE_ROWS = 256
OK, BAD = N.LO_OK, N.LO_ERR_INVALID
CHARS = np.frombuffer(b"12345678", np.uint8)
NAN_BITS = 0x7FF8000000000000


def _off(*v):
    return np.array(v, np.int64)


def _validity(mask=False, bitmap=False, bit_offset=0):
    v = N.Validity()
    if mask:
        v.mask = CHARS.ctypes.data
    if bitmap:
        v.bitmap, v.bit_offset = CHARS.ctypes.data, bit_offset
    return v


# case: (chars, offsets, n, validity, expected return code per entry point; None where the entry point takes no validity
# or would read past the offsets)
BAD_INPUTS = {
    "null_offsets": (CHARS, None, 2, None, (BAD, BAD, BAD, BAD)),
    "null_chars_with_bytes": (None, _off(0, 1, 2), 2, None, (BAD, BAD, BAD, BAD)),
    "last_offset_before_the_first": (CHARS, _off(4, 5, 2), 2, None, (BAD, BAD, BAD, BAD)),
    "one_descending_pair": (CHARS, _off(0, 3, 1, 4), 3, None, (BAD, BAD, OK, BAD)),
    "first_offset_not_zero": (CHARS, _off(2, 3, 5), 2, None, (BAD, OK, OK, OK)),
    "mask_and_bitmap": (CHARS, _off(0, 1, 2), 2, _validity(mask=True, bitmap=True), (None, None, BAD, BAD)),
    "negative_bit_offset": (CHARS, _off(0, 1, 2), 2, _validity(bitmap=True, bit_offset=-1), (None, None, BAD, BAD)),
    "2^31_rows_two_offsets": (CHARS, _off(0, 0), 2 ** 31, None, (BAD, None, BAD, BAD)),
    "no_rows_null_offsets": (CHARS, None, 0, None, (OK, OK, OK, BAD)),
}


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _call(engine, table, entry, chars, offsets, n, validity):
    """(return code, lo_host_timing, what the call produced): groups (rep rows, counts) / (values, status) / the
    lo_parse_summary / (groups, null cells) of the resident column, which is freed again."""
    from learningorchestra_b200.engine import DeviceText
    lib, ctx, t = engine._lib, engine._ctx, N.HostTiming()
    v = C.byref(validity) if validity is not None else None
    if entry == "value_counts_str":
        cap = min(max(n, 1), TABLE_ROWS)
        rows, counts, nd = np.zeros(cap, np.int64), np.zeros(cap, np.uint64), C.c_int64(-1)
        rc = lib.lo_value_counts_str_host(ctx, _ptr(chars), _ptr(offsets), n, _ptr(rows), _ptr(counts), cap, C.byref(nd),
                                          C.byref(t))
        return rc, t, (rows[:max(nd.value, 0)], counts[:max(nd.value, 0)])
    if entry == "parse_number":
        values, status = np.zeros(max(n, 1), np.float64), np.zeros(max(n, 1), np.uint8)
        rc = lib.lo_parse_number_host(ctx, _ptr(chars), _ptr(offsets), n, _ptr(values), _ptr(status), C.byref(t))
        return rc, t, (values[:n], status[:n])
    if entry == "parse_number_to_table":
        s = N.ParseSummary()
        rc = lib.lo_parse_number_to_table(ctx, _ptr(chars), _ptr(offsets), v, n, table._h, 0, 0, C.byref(s), C.byref(t))
        return rc, t, s
    h = C.c_void_p()
    rc = lib.lo_text_upload(ctx, _ptr(chars), _ptr(offsets), v, n, C.byref(h), C.byref(t))
    if rc != OK:
        return rc, t, None
    text = DeviceText(engine, h, None)
    try:
        return rc, t, (engine.value_counts_text(text), text.nulls)
    finally:
        text.free()


@pytest.fixture(scope="module")
def table(engine):
    t = engine.table("f64", TABLE_ROWS, 1)
    yield t
    t.free()


@pytest.mark.parametrize("case", list(BAD_INPUTS))
def test_malformed_text_arguments(engine, table, case):
    chars, offsets, n, validity, expected = BAD_INPUTS[case]
    for entry, rc_expected in zip(ENTRIES, expected):
        if rc_expected is None:
            continue
        before = engine.launch_count
        rc, _, out = _call(engine, table, entry, chars, offsets, n, validity)
        assert rc == rc_expected, (case, entry, engine._lib.lo_last_error())
        if rc != OK:
            assert engine.launch_count == before, (case, entry)
        if case == "one_descending_pair" and entry == "parse_number_to_table":
            assert (out.first_invalid, out.first_unsupported) == (-1, 1)


def _float_bits(cell):
    return int(np.float64(float(cell)).view(np.uint64))


def test_a_sliced_column_with_nulls_through_every_entry_point(engine, table):
    import pyarrow as pa
    rng = np.random.default_rng(11)
    words = ["0", "1", "-7", "2.5", "1e3", "", "0.125", "42", "-0.0", " 3.75 "]
    cells = [None if i % 7 == 3 else words[j] for i, j in enumerate(rng.integers(0, len(words), 300))]
    arr = pa.array(cells, type=pa.large_string()).slice(13, 200)
    chars, offsets, (bitmap, bit_offset) = text_buffers(arr)
    n, vals = len(arr), arr.to_pylist()
    assert bit_offset % 8 != 0 and offsets[0] != 0 and arr.null_count
    validity = N.Validity()
    validity.bitmap, validity.bit_offset = bitmap.ctypes.data, bit_offset
    raw = [bytes(chars[offsets[i]:offsets[i + 1]]) for i in range(n)]
    span = int(offsets[n] - offsets[0])
    valid_bytes = ((bit_offset + n - 1) >> 3) - (bit_offset >> 3) + 1

    # the host group-by: no validity, offsets from 0; a null cell counts as its (empty) bytes
    rc, t, (rows, counts) = _call(engine, table, "value_counts_str", chars[offsets[0]:], offsets - offsets[0], n, None)
    assert rc == OK and t.h2d_bytes == span + 8 * (n + 1)
    assert {raw[int(r)]: int(c) for r, c in zip(rows, counts)} == dict(Counter(raw))

    rc, t, (values, status) = _call(engine, table, "parse_number", chars, offsets, n, None)
    assert rc == OK and t.h2d_bytes == span + 8 * (n + 1)
    for i, b in enumerate(raw):
        if b == b"":
            assert status[i] == N.LO_NUM_EMPTY, i
            continue
        v = float(b)
        assert status[i] == (N.LO_NUM_INTEGER if v.is_integer() else N.LO_NUM_FLOAT), i
        assert int(values[i:i + 1].view(np.uint64)[0]) == _float_bits(b), i

    rc, t, s = _call(engine, table, "parse_number_to_table", chars, offsets, n, validity)
    assert rc == OK and t.h2d_bytes == span + 8 * (n + 1) + valid_bytes
    present = [c for c in vals if c not in (None, "")]
    assert (s.first_invalid, s.first_unsupported, s.nulls) == (-1, -1, n - len(present))
    assert bool(s.all_integer) == all(float(c).is_integer() for c in present)
    got = table.to_numpy(0, 0, n).view(np.uint64).tolist()
    assert got == [NAN_BITS if c in (None, "") else _float_bits(c) for c in vals]

    rc, t, ((rows, counts), nulls) = _call(engine, table, "text_upload", chars, offsets, n, validity)
    assert rc == OK and t.h2d_bytes == span + 8 * (n + 1) + valid_bytes
    assert nulls == arr.null_count
    assert {vals[int(r)]: int(c) for r, c in zip(rows, counts)} == dict(Counter(c for c in vals if c is not None))
