"""GPU: the "number" cast's parser (csrc/parse_number.cuh in k_parse_number / k_parse_number_to_col) against CPython's
own float() on every entry point that runs it — lo_parse_number_host, lo_parse_number_to_table (every validity form,
shard cuts) and lo_parse_text_to_table — over the corpus test_parse_cpu.py checks on the CPU, the 1 MiB length limit
and the summary's reductions across grid sweeps; then the resident "string" cast (lo_format_table_to_text) with its
valid / is_int flags as byte masks, bitmaps at any bit offset and NULL, against repr(float) / str(int).

The device build runs code the CPU harness does not (__umul64hi, __clzll, the power-of-five table in device memory,
the slow path's big integers in local memory), and it reads the staged chars with nothing after the last cell, so
every expected value here comes from Python, never from another GPU route."""
import ctypes as C
import re

import numpy as np
import pyarrow as pa
import pytest

from learningorchestra_b200 import _native as N
from learningorchestra_b200.columnar import ascii_number_text, text_buffers
from learningorchestra_b200.engine import DeviceText
from learningorchestra_b200.sharding import ShardedEngine, combine_parse_summaries
from test_format_cpu import expected as format_expected
from test_gpu_format import _value_sets
from test_parse_cpu import (EMPTY, FLOAT, INTEGER, INVALID, UNSUPPORTED, expected, grammar_cases, halfway_and_long_digits,
                            long_cells, random_short_decimals, unicode_cells)

pytestmark = pytest.mark.gpu
NAN = 0x7FF8000000000000                 # what a null or "" cell stores
MAX_LEN = 1 << 20                        # num::kMaxLen
BLOCK = 128                              # the parse and format kernels' block size; the grid is capped at 16 blocks per SM


def test_status_codes_are_the_cpu_harness_codes():
    assert (N.LO_NUM_FLOAT, N.LO_NUM_INTEGER, N.LO_NUM_EMPTY, N.LO_NUM_INVALID, N.LO_NUM_UNSUPPORTED) == \
        (FLOAT, INTEGER, EMPTY, INVALID, UNSUPPORTED)


# ---- Python's answers -------------------------------------------------------------------------------------------
def _expect(cells):
    """(status uint8[n], bits uint64[n]) of expected() per cell; bytes cells are decoded first."""
    out = [expected(c.decode("utf-8") if isinstance(c, bytes) else c) for c in cells]
    return np.array([s for s, _ in out], np.uint8), np.array([b for _, b in out], np.uint64)


def _summary(status, null):
    """The summary lo_parse_number_to_table must report for cells of ``status`` with ``null`` (bool) rows null."""
    live = ~null
    invalid = np.flatnonzero(live & (status == INVALID))
    unsupported = np.flatnonzero(live & (status == UNSUPPORTED))
    return {"first_invalid": int(invalid[0]) if invalid.size else None,
            "first_unsupported": int(unsupported[0]) if unsupported.size else None,
            "nulls": int((null | (status == EMPTY)).sum()),
            "integer": bool(np.all(~live | (status == INTEGER) | (status == EMPTY)))}


def _same_summary(got, want, what):
    assert {k: got[k] for k in want} == want, what


def _column_bits(status, bits, null):
    """What the f64 column holds: float()'s bits for the cells it accepts, the canonical NaN for null and "" cells.
    Rows float() refuses are None: the call reports them and the caller fails, so their bits are not specified."""
    out = np.where(null | (status == EMPTY), np.uint64(NAN), bits)
    keep = null | (status == EMPTY) | (status == FLOAT) | (status == INTEGER)
    return out, keep


def _assert_bits(got, want, keep, cells, what):
    bad = np.flatnonzero(keep & (got != want))
    if bad.size:
        i = int(bad[0])
        cell = cells[i] if cells is not None else None
        pytest.fail(f"{what}: {bad.size} rows differ, first row {i} {str(cell)[:80]!r}: {hex(int(got[i]))} != {hex(int(want[i]))}")


# ---- the slow path: restated from parse_number() ---------------------------------------------------------------
_DECIMAL = re.compile(r"[+-]?(\d*)(?:\.(\d*))?(?:[eE]([+-]?\d+))?", re.ASCII)


def _takes_slow_path(cell: str) -> bool:
    """True when parse_number() decides ``cell`` with the big-integer comparison: more than 19 significant digits with a
    nonzero digit dropped, and the truncated significand w and w + 1 (at w's decimal exponent q) round to different
    doubles."""
    try:
        float(cell)
    except ValueError:
        return False
    m = _DECIMAL.fullmatch(cell.strip(" \t\n\v\f\r").replace("_", ""))
    if not m:                                        # inf / nan
        return False
    ip, fp, exp = m.group(1), m.group(2) or "", m.group(3) or "0"
    digits = (ip + fp).lstrip("0")
    if len(digits) <= 19 or not digits[19:].strip("0"):
        return False
    w, q = int(digits[:19]), int(exp) - len(fp) + len(digits) - 19
    return float(f"{w}e{q}") != float(f"{w + 1}e{q}")


# ---- the corpus ---------------------------------------------------------------------------------------------------
class Corpus:
    """test_parse_cpu.py's cells, normalised by the packer's rule (what float(str) does first), in one column: the short
    decimals, the halfway and long-digit cells, the long cells, then the grammar and Unicode cases (whose invalid cells
    come last, so the first bad row is far from row 0)."""

    def __init__(self):
        raw = random_short_decimals() + halfway_and_long_digits() + long_cells() + grammar_cases() + unicode_cells()
        self.cells = [ascii_number_text(c) for c in raw]
        self.status, self.bits = _expect(raw)          # float(str) of the original: the normalisation is part of it
        self.arr = pa.array(self.cells, type=pa.large_string())
        self.chars, self.offsets, _ = text_buffers(self.arr)


@pytest.fixture(scope="module")
def corpus():
    return Corpus()


def test_the_corpus_reaches_the_slow_path(corpus):
    slow = sum(map(_takes_slow_path, corpus.cells))
    assert slow >= 4000, slow


def test_the_slow_path_restatement():
    assert _takes_slow_path("1.00000000000000011102230246251565404236316680908203125")          # 1 + 2^-53: a tie
    assert _takes_slow_path("  -9007199254740993.000000000000000000001e0 ")                      # 2^53 + 1, nudged up
    assert not _takes_slow_path("1.000000000000000000000000")          # trailing zeros drop nothing
    assert not _takes_slow_path("12345678901234567891234")             # w and w + 1 round alike
    assert not _takes_slow_path("0.1") and not _takes_slow_path("abc") and not _takes_slow_path("1e5")


# ---- lo_parse_number_host ---------------------------------------------------------------------------------------
def test_packed_route_equals_float(engine, corpus):
    values, status = engine.parse_number_packed(corpus.chars, corpus.offsets)
    bad = np.flatnonzero(status != corpus.status)
    assert not bad.size, [(corpus.cells[i][:60], int(status[i]), int(corpus.status[i])) for i in bad[:5]]
    number = (status == FLOAT) | (status == INTEGER)
    _assert_bits(values.view(np.uint64), corpus.bits, number, corpus.cells, "packed")
    # a slice of the same column: offsets[0] != 0, rebased on the host
    sl = corpus.arr.slice(299_990, 26_700)
    chars, offsets, _ = text_buffers(sl)
    assert offsets[0] != 0
    values, status = engine.parse_number_packed(chars, offsets)
    assert np.array_equal(status, corpus.status[299_990:299_990 + 26_700])
    _assert_bits(values.view(np.uint64), corpus.bits[299_990:299_990 + 26_700], number[299_990:299_990 + 26_700],
                 corpus.cells[299_990:], "packed slice")


def test_raw_non_ascii_cells_are_unsupported(engine):
    from learningorchestra_b200.columnar import pack_cells
    raw = grammar_cases() + unicode_cells()
    values, status = engine.parse_number_packed(*pack_cells(raw))
    for c, s in zip(raw, status.tolist()):
        assert s == UNSUPPORTED if not c.isascii() else s == expected(c)[0], (c, s)


# ---- lo_parse_number_to_table: every validity form ---------------------------------------------------------------
def _with_nulls(corpus, every=29):
    """The corpus with a null cell after every ``every`` cells; a null cell's slot holds text that would be invalid
    ("x") or would break the integer flag ("2.5") if it were read.  Returns (cells, chars, offsets, null, status, bits)."""
    cells, null = [], []
    for i, c in enumerate(corpus.cells):
        if i % every == 3:
            cells.append("x" if i % 2 else "2.5")
            null.append(True)
        cells.append(c)
        null.append(False)
    null = np.array(null)
    status, bits = np.empty(len(cells), np.uint8), np.empty(len(cells), np.uint64)
    status[~null], bits[~null] = corpus.status, corpus.bits
    status[null], bits[null] = EMPTY, NAN          # what the summary and the column make of a null
    arr = pa.array(cells, type=pa.large_string())
    chars, offsets, _ = text_buffers(arr)
    return cells, chars, offsets, null, status, bits


def _bitmap(valid, bit_offset, seed):
    """An Arrow validity bitmap of ``valid`` starting at ``bit_offset``, the bits before and after it random."""
    rng = np.random.default_rng(seed)
    pad = rng.integers(0, 2, bit_offset + 16).astype(bool)
    bits = np.concatenate([pad[:bit_offset], valid, pad[bit_offset:]])
    return np.packbits(bits, bitorder="little")


def _parse_into(engine, chars, offsets, nulls):
    t = engine.table("f64", offsets.shape[0] - 1, 1)
    try:
        s = engine.parse_number_into(t, 0, chars, offsets, nulls)
        return t.to_numpy(0).view(np.uint64).copy(), s
    finally:
        t.free()


@pytest.fixture(scope="module")
def nulled(corpus):
    return _with_nulls(corpus)


def _null_forms(null):
    """(name, nulls argument) for every form parse_number_into takes: a bool mask, and Arrow bitmaps at bit offsets
    1 to 7 and 13."""
    yield "mask", null
    for k in list(range(1, 8)) + [13]:
        yield f"bitmap+{k}", (_bitmap(~null, k, k), k)


def test_to_table_equals_float_for_every_validity_form(engine, nulled):
    cells, chars, offsets, null, status, bits = nulled
    want, keep = _column_bits(status, bits, null)
    want_summary = _summary(status, null)
    assert want_summary["first_invalid"] is not None and want_summary["first_invalid"] > 300_000
    for name, nulls in _null_forms(null):
        got, s = _parse_into(engine, chars, offsets, nulls)
        _assert_bits(got, want, keep, cells, name)
        _same_summary(s, want_summary, name)
    # no validity: the null rows' slots are read as cells
    st_slots, bits_slots = _expect(cells)
    none = np.zeros(len(cells), bool)
    want, keep = _column_bits(st_slots, bits_slots, none)
    got, s = _parse_into(engine, chars, offsets, None)
    _assert_bits(got, want, keep, cells, "no validity")
    _same_summary(s, _summary(st_slots, none), "no validity")
    assert s["first_invalid"] == 3 and null[3] and cells[3] == "x"        # the first null slot


def test_to_table_on_a_sliced_arrow_array(engine, nulled):
    cells, _, _, null, status, bits = nulled
    arr = pa.array([None if z else c for c, z in zip(cells, null)], type=pa.large_string())
    for start, length in ((5, 300_001), (299_997, len(cells) - 299_997), (len(cells) - 1, 1)):
        sl = arr.slice(start, length)
        chars, offsets, validity = text_buffers(sl)
        assert offsets[0] != 0 and (validity is None or validity[1] == start)
        got, s = _parse_into(engine, chars, offsets, validity)
        sn, sst = null[start:start + length], status[start:start + length]
        want, keep = _column_bits(sst, bits[start:start + length], sn)
        _assert_bits(got, want, keep, cells[start:], f"slice {start}")
        _same_summary(s, _summary(sst, sn), f"slice {start}")


# ---- shard cuts -------------------------------------------------------------------------------------------------
def _shard_nulls(nulls, off, nr):
    """The nulls of rows [off, off + nr) as ShardedEngine.parse_number_into hands them to a member."""
    if nulls is None:
        return None
    if isinstance(nulls, tuple):
        return nulls[0], int(nulls[1]) + off
    return nulls[off:off + nr]


def test_shard_cuts_merge_to_the_single_call(engine, nulled):
    cells, chars, offsets, null, status, bits = nulled
    n = len(cells)
    cuts = [0, 1, 4099, 77_777, 300_003, 310_001, n - 3, n]
    want, keep = _column_bits(status, bits, null)
    want_summary = _summary(status, null)
    for name, nulls in [("none", None)] + list(_null_forms(null))[::4]:
        single_bits, single = _parse_into(engine, chars, offsets, nulls)
        parts, pieces = [], []
        for b, e in zip(cuts[:-1], cuts[1:]):
            got, s = _parse_into(engine, chars, offsets[b:e + 1], _shard_nulls(nulls, b, e - b))
            parts.append(s)
            pieces.append(got)
        merged = combine_parse_summaries(parts, cuts[:-1])
        assert np.array_equal(np.concatenate(pieces), single_bits), name
        _same_summary(merged, {k: single[k] for k in ("first_invalid", "first_unsupported", "nulls", "integer")}, name)
        if nulls is not None:
            _assert_bits(single_bits, want, keep, cells, name)
            _same_summary(merged, want_summary, name)
    # a bad cell in the last shard only: its row comes back global
    row = max(r for r in range(n - 3, n) if not null[r])
    bad = list(cells)
    bad[row] = "é"
    tail_chars, tail_offsets, _ = text_buffers(pa.array(bad, type=pa.large_string()))
    parts = [_parse_into(engine, tail_chars, tail_offsets[b:e + 1], _shard_nulls(null, b, e - b))[1]
             for b, e in zip(cuts[:-1], cuts[1:])]
    assert combine_parse_summaries(parts, cuts[:-1])["first_unsupported"] == row


def test_sharded_engine_over_every_visible_gpu(engine, nulled):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: the shard cuts above are the sharded parse's slices")
    cells, chars, offsets, null, status, bits = nulled
    want, keep = _column_bits(status, bits, null)
    with ShardedEngine.local() as sh:
        for nulls in (null, (_bitmap(~null, 5, 5), 5)):
            t = sh.table("f64", len(cells), 1)
            try:
                s = sh.parse_number_into(t, 0, chars, offsets, nulls)
                got = np.concatenate([p.to_numpy(0).view(np.uint64) for p in t.shards])
            finally:
                t.free()
            _assert_bits(got, want, keep, cells, "sharded")
            _same_summary(s, _summary(status, null), "sharded")


# ---- lo_parse_text_to_table -------------------------------------------------------------------------------------
def test_resident_text_route_equals_float(engine, nulled):
    cells, _, _, null, status, bits = nulled
    full = pa.array([None if z else c for c, z in zip(cells, null)], type=pa.large_string())
    for start, length in ((0, len(cells)), (3, len(cells) - 10)):       # a slice: offsets rebased, bitmap from bit 3
        arr = full.slice(start, length)
        text = engine.text(arr)
        t = engine.table("f64", length, 1)
        try:
            s = engine.parse_text_into(t, 0, text)
            got = t.to_numpy(0).view(np.uint64)
        finally:
            t.free()
            text.free()
        sn, sst = null[start:start + length], status[start:start + length]
        want, keep = _column_bits(sst, bits[start:start + length], sn)
        _assert_bits(got, want, keep, cells[start:], f"text {start}")
        _same_summary(s, _summary(sst, sn), f"text {start}")


# ---- the 1 MiB limit --------------------------------------------------------------------------------------------
def _limit_cells():
    """Cells of exactly 1 MiB whose answer rests on a digit past the 800th, one that is mostly whitespace, one of
    1 MiB + 1 bytes, and short cells around them."""
    tie = "1." + str(5 ** 53).rjust(53, "0")                 # 1 + 2^-53: ties to 1.0
    sub = "0." + str(5 ** 1075).rjust(1075, "0")             # 2^-1075: ties to 0.0
    assert len(sub) > 800
    pad = lambda s, tail: s + "0" * (MAX_LEN - len(s) - len(tail)) + tail      # noqa: E731
    cells = ["1.5", pad(tie, "1"), pad(tie, "0"), "-7", pad(sub, "1e0"), pad(sub, "e0"),
             " " * (MAX_LEN - 5) + "1e5\t\n", "9" * (MAX_LEN + 1), "2"]
    assert [len(c) for c in cells[1:3] + cells[4:7]] == [MAX_LEN] * 5 and len(cells[7]) == MAX_LEN + 1
    return cells


def test_cells_of_one_mib_on_every_entry_point(engine):
    cells = _limit_cells()
    status, bits = _expect(cells)
    status[7] = UNSUPPORTED                             # float() reads it; the device does not, and says so
    assert [float(c) for c in cells[1:3]] == [1.0000000000000002, 1.0] and [float(c) for c in cells[4:6]] == [5e-324, 0.0]
    arr = pa.array(cells, type=pa.large_string())
    chars, offsets, _ = text_buffers(arr)
    values, st = engine.parse_number_packed(chars, offsets)
    assert st.tolist() == status.tolist()
    ok = (status == FLOAT) | (status == INTEGER)
    assert np.array_equal(values.view(np.uint64)[ok], bits[ok])
    null = np.zeros(len(cells), bool)
    want, keep = _column_bits(status, bits, null)
    got, s = _parse_into(engine, chars, offsets, None)
    _assert_bits(got, want, keep, None, "to_table")
    _same_summary(s, _summary(status, null), "to_table")
    assert s["first_unsupported"] == 7
    text = engine.text(arr)
    t = engine.table("f64", len(cells), 1)
    try:
        s = engine.parse_text_into(t, 0, text)
        _assert_bits(t.to_numpy(0).view(np.uint64), want, keep, None, "text")
    finally:
        t.free()
        text.free()
    _same_summary(s, _summary(status, null), "text")


# ---- the summary across grid sweeps -----------------------------------------------------------------------------
def _grid_threads(engine, n):
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return min((n + BLOCK - 1) // BLOCK, sm * 16) * BLOCK


def _placements(n, threads):
    """{row: cell} sets of invalid ("x") and unsupported ("é") cells: rows 0 and n - 1, lane 31, and a smallest bad row
    in the last block of sweep 0 while block 0 holds a larger one in sweep 1 (and the same a sweep later)."""
    last_block_lane31 = threads - BLOCK + 31
    return [{}, {n - 1: "2.5"},                                             # only the integer flag changes
            {0: "x", n - 1: "é"},
            {31: "é", n - 1: "x", n - 2: "é"},
            {last_block_lane31: "x", threads + 3: "x", last_block_lane31 - 64: "é", 2 * threads + 1: "é"},
            {threads + last_block_lane31: "x", 2 * threads + 3: "x", n - 1: "x", 2 * threads - 1: "é", 2 * threads + 32: "é"}]


@pytest.fixture(scope="module")
def million(engine):
    """1 000 003 integer cells, every 11th "" and every 7th null (its slot "0.5"), none of the placed rows null; the
    placements for the kernel's sweep size."""
    n = 1_000_003
    threads = _grid_threads(engine, n)
    assert n >= 3 * threads, threads                     # every thread loops at least three times
    places = _placements(n, threads)
    cells = [str(i * 7 - 3_000_000) for i in range(n)]
    for i in range(0, n, 11):
        cells[i] = ""
    null = np.zeros(n, bool)
    null[3::7] = True
    null[[r for p in places for r in p]] = False
    for i in np.flatnonzero(null):
        cells[i] = "0.5"
    status, bits = _expect(cells)
    return cells, null, status, bits, places


def test_summary_reductions_across_million_cell_sweeps(engine, million):
    cells, null, status, bits, places = million
    n = len(cells)
    for k, place in enumerate(places):
        c, st, bt = list(cells), status.copy(), bits.copy()
        for row, cell in place.items():
            c[row] = cell
            st[row], bt[row] = (UNSUPPORTED, 0) if cell == "é" else expected(cell)     # a raw byte >= 0x80
        want_summary = _summary(st, null)
        want, keep = _column_bits(st, bt, null)
        chars, offsets, _ = text_buffers(pa.array(c, type=pa.large_string()))
        nulls = null if k % 2 else (_bitmap(~null, k, k), k)
        got, s = _parse_into(engine, chars, offsets, nulls)
        _same_summary(s, want_summary, (k, place))
        _assert_bits(got, want, keep, None, str(place))
        if k in (0, 4):          # the resident text route: the same kernel over a column uploaded once
            text = engine.text(pa.array([None if z else v for v, z in zip(c, null)], type=pa.large_string()))
            t = engine.table("f64", n, 1)
            try:
                s = engine.parse_text_into(t, 0, text)
                _assert_bits(t.to_numpy(0).view(np.uint64), want, keep, None, f"text {place}")
            finally:
                t.free()
                text.free()
            _same_summary(s, want_summary, ("text", place))
    assert _summary(status, null)["integer"] is True and _summary(status, null)["nulls"] > n // 7


# ---- lo_format_table_to_text: the flag forms --------------------------------------------------------------------
def _flag(flags, form, seed):
    """(lo_validity or None, the array it points into) of bool ``flags`` as ``form``: "mask" (random nonzero bytes
    for True), an int bit offset (an Arrow bitmap), or None (NULL)."""
    if form is None:
        return None, None
    v = N.Validity()
    if form == "mask":
        rng = np.random.default_rng(seed)
        keep = np.where(flags, rng.integers(1, 256, flags.shape[0]), 0).astype(np.uint8)
        v.mask = keep.ctypes.data
    else:
        keep = _bitmap(flags, form, seed)
        v.bitmap, v.bit_offset = keep.ctypes.data, form
    return v, keep


def _format(engine, values, valid_form, is_int_form, valid, is_int, seed=0):
    """lo_format_table_to_text of ``values`` through the C ABI: (rc, offsets, chars) read back with download_text."""
    table = engine.table_from_numpy([np.ascontiguousarray(values, np.float64)]) if len(values) else engine.table("f64", 0, 1)
    (v, _kv), (i, _ki) = _flag(valid, valid_form, seed), _flag(is_int, is_int_form, seed + 1)
    h, t = C.c_void_p(), N.HostTiming()
    try:
        rc = engine._lib.lo_format_table_to_text(engine._ctx, table._h, 0, C.byref(v) if v is not None else None,
                                                 C.byref(i) if i is not None else None, C.byref(h), C.byref(t))
        if rc != N.LO_OK:
            return rc, None, None
        text = DeviceText(engine, h, None)
        try:
            offsets, chars = engine.download_text(text)
        finally:
            text.free()
        return rc, offsets, chars[:offsets[-1]]
    finally:
        table.free()


class _Texts:
    """repr(float) and str(int) of every value, each computed once."""

    def __init__(self, values):
        self.float = [format_expected(v, FLOAT) for v in values.tolist()]
        ok = np.isfinite(values) & (values == np.floor(np.where(np.isfinite(values), values, 0)))
        self.integral = ok
        self.int = [format_expected(v, INTEGER) if z else None for v, z in zip(values.tolist(), ok.tolist())]

    def want(self, valid, is_int):
        out = []
        for f, it, a, b in zip(self.float, self.int, valid.tolist(), is_int.tolist()):
            out.append("" if not a else it if b else f)
        return out


def _check_text(offsets, chars, want, what):
    lens = np.fromiter((len(w) for w in want), np.int64, len(want))
    assert offsets[0] == 0 and np.array_equal(np.diff(offsets), lens), what
    if chars.tobytes() != "".join(want).encode():
        for i, w in enumerate(want):
            assert chars[offsets[i]:offsets[i + 1]].tobytes().decode() == w, (what, i, w)


@pytest.fixture(scope="module")
def format_rows():
    """_value_sets() and a million random bit patterns: valid ~90 %, is_int on about half of the integral values;
    row 0 not valid, row 1 an integer, the last row a float."""
    values, status = _value_sets()
    rng = np.random.default_rng(20261017)
    rand = rng.integers(0, 2 ** 64, size=1_000_000, dtype=np.uint64).view(np.float64)
    values = np.concatenate([np.array([2.5, 3.0]), values, rand, np.array([0.1])])
    texts = _Texts(values)
    valid = np.concatenate([[False, True], status != EMPTY, rng.random(rand.size) < 0.9, [True]])
    is_int = np.concatenate([[False, True], status == INTEGER, texts.integral[2 + status.size:-1] & (rng.random(rand.size) < 0.5),
                             [False]])
    assert not np.any(is_int & ~texts.integral)
    return values, valid, is_int, texts


_FORMS = [("mask", "mask")] + [(k, k) for k in list(range(8)) + [13]] + \
    [(None, 3), (6, None), (None, None), ("mask", 5), (13, "mask"), (None, "mask")]


def test_format_flag_forms_equal_repr_on_a_million_rows(engine, format_rows):
    values, valid, is_int, texts = format_rows
    n = values.shape[0]
    for vf, f in _FORMS:
        v = valid if vf is not None else np.ones(n, bool)          # NULL valid: every row valid
        i = is_int if f is not None else np.zeros(n, bool)         # NULL is_int: no row an integer
        rc, offsets, chars = _format(engine, values, vf, f, valid, is_int, seed=10 * _FORMS.index((vf, f)))
        assert rc == N.LO_OK, (vf, f, N.load().lo_last_error())
        _check_text(offsets, chars, texts.want(v, i), (vf, f))


def test_format_one_row_and_zero_rows(engine):
    for value, valid, is_int in ((2.5, True, False), (3.0, True, True), (3.0, False, True), (1e22, True, True),
                                 (1e22, True, False), (-0.0, True, False), (-0.0, True, True)):
        for vf, f in _FORMS:
            rc, offsets, chars = _format(engine, np.array([value]), vf, f, np.array([valid]), np.array([is_int]))
            shown, as_int = valid or vf is None, is_int and f is not None      # NULL: every row valid, none an integer
            exp = format_expected(value, INTEGER if as_int else FLOAT) if shown else ""
            assert rc == N.LO_OK and offsets.tolist() == [0, len(exp)] and chars.tobytes().decode() == exp, (value, vf, f)
    for vf, f in _FORMS:
        rc, offsets, chars = _format(engine, np.zeros(0), vf, f, np.zeros(0, bool), np.zeros(0, bool))
        assert rc == N.LO_OK and offsets.tolist() == [0] and chars.size == 0, (vf, f)


def test_format_refusal_names_the_lowest_of_a_million_rows(engine):
    n = 1_000_003
    threads = _grid_threads(engine, n)
    low = threads - BLOCK + 31                      # the last block of sweep 0, lane 31
    high = threads + 3                              # block 0, sweep 1: a lower block holding a larger row
    values = np.arange(n, dtype=np.float64)
    values[[low, high]] = 0.5
    valid, is_int = np.ones(n, bool), np.ones(n, bool)
    for forms in (("mask", "mask"), (None, 5), (2, 13)):
        rc, _, _ = _format(engine, values, *forms, valid, is_int)
        msg = N.load().lo_last_error().decode()
        assert rc == N.LO_ERR_INVALID and f"row {low}:" in msg, (forms, msg)
    # a non-integral row that is not valid, or not flagged, is no refusal
    valid[low] = False
    is_int[high] = False
    rc, offsets, chars = _format(engine, values, "mask", 7, valid, is_int)
    assert rc == N.LO_OK and chars[offsets[high]:offsets[high + 1]].tobytes() == b"0.5" and offsets[low] == offsets[low + 1]
