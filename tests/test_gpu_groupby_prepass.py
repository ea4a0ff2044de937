"""GPU: the kernels behind the endpoints users call, at the inputs where a hash table or a reduction goes wrong.

* numeric ``$group`` (``k_hash_count_f64``): every NaN and zero bit pattern, keys one ulp apart, keys chosen so that every
  insert starts at the table's last slot and wraps, the table-size boundaries, a grid-stride column, the capacity contract;
* text ``$group`` (``k_hash_count_str``): cell pairs whose 33-bit slot tags and start slots collide
  (tests/golden/hash_collisions.json), byte-level edge cells, the row limit, a sliced Arrow column;
* the range pre-pass (``k_minmax_cast``) through the host pipeline, a resident table and a sharded table;
* every ``*_host`` entry point cut into more chunks than the pipeline has staging slots;
* binned histograms without ``range`` whose plain [min, max] the kernels would reject (``auto_range``).

Every expected value comes from a plain reference: ``collections.Counter`` over ``oracle.rsem.group_key``, numpy over
``bn.cast_f64_f32``, ``bn.project_cast_hist`` / ``np.bincount``; floats are compared by their bits."""
import ctypes as C
import json
from collections import Counter
from pathlib import Path

import numpy as np
import pytest
from werkzeug.test import Client

from edge_values import F32_MAX, NAN_BITS
from edge_values import f64 as _f64
from edge_values import prepass_columns as _prepass_columns
from edge_values import ref_minmax as _ref_minmax
from learningorchestra_b200 import _native as N
from learningorchestra_b200 import server, utils
from oracle import bsem_numpy as bn
from oracle import rsem

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"


def _table_slots(n: int) -> int:
    """Slots of the group-by hash table for n rows: max(1024, the smallest power of two >= 2n)."""
    s = 1024
    while s < 2 * n:
        s <<= 1
    return s


# ---- numeric $group ---------------------------------------------------------------------------------------------
ZERO_BITS = [0x0000000000000000, 0x8000000000000000]


def _special_f64():
    one_ulp = [1.0, 0.1, -3.5, 1e300, 2.0 ** -1022, 123456.789]
    vals = [np.inf, -np.inf, 5e-324, -5e-324, np.finfo(np.float64).max, -np.finfo(np.float64).max, 2.0 ** 53,
            2.0 ** 53 + 2, 2.0 ** 53 - 1, -(2.0 ** 53)]
    for v in one_ulp:
        vals += [v, float(np.nextafter(v, np.inf))]
    return np.concatenate([_f64(NAN_BITS), _f64(ZERO_BITS), np.array(vals)])


def _check_value_counts_f64(engine, x):
    keys, counts = engine.value_counts_f64_host(x)
    kb = keys.view(np.uint64)
    # the keys the kernel reports are canonical: one NaN pattern, no -0.0
    assert not any(int(b) in NAN_BITS[1:] for b in kb) and 0x8000000000000000 not in kb.tolist()
    assert np.isnan(keys).sum() <= 1 and (kb[np.isnan(keys)] == 0x7FF8000000000000).all()
    got = {rsem.group_key(float(k)): int(c) for k, c in zip(keys, counts)}
    assert len(got) == len(keys)                               # no group reported twice
    # reference: exact bit patterns counted by numpy, merged under MongoDB's equality
    u, uc = np.unique(x.view(np.uint64), return_counts=True)
    exp = Counter()
    for b, c in zip(u.view(np.float64), uc):
        exp[rsem.group_key(float(b))] += int(c)
    assert got == dict(exp)
    assert int(counts.sum()) == x.size


def test_value_counts_f64_nan_and_zero_bit_patterns(engine):
    rng = np.random.default_rng(21)
    sp = _special_f64()
    x = np.concatenate([np.repeat(sp, rng.integers(1, 40, sp.size)), sp])
    rng.shuffle(x)
    _check_value_counts_f64(engine, x)
    keys, counts = engine.value_counts_f64_host(x)
    by_bits = dict(zip(keys.view(np.uint64).tolist(), counts.tolist()))
    nan_rows = int(np.isnan(x).sum())
    zero_rows = int((x == 0).sum())
    assert by_bits[0x7FF8000000000000] == nan_rows and by_bits[0] == zero_rows
    assert len(keys) == sp.size - len(NAN_BITS) - len(ZERO_BITS) + 2


@pytest.mark.parametrize("n", [1, 31, 32, 33, 512, 513])
def test_value_counts_f64_table_size_edges(engine, n):
    rng = np.random.default_rng(n)
    pool = np.concatenate([_special_f64(), rng.integers(-20, 20, 40).astype(np.float64) * 0.25])
    x = pool[rng.integers(0, pool.size, n)]
    if n == 1:
        x = _f64([0xFFFFFFFFFFFFFFFF])                         # the table's empty-slot marker as the only value
    _check_value_counts_f64(engine, x)


def test_value_counts_f64_grid_stride_column(engine):
    rng = np.random.default_rng(4)
    n = 3_000_000
    x = rng.integers(-300_000, 300_000, n).astype(np.float64) * 0.5
    hit = rng.random(n) < 0.01
    x[hit] = _special_f64()[rng.integers(0, _special_f64().size, int(hit.sum()))]
    _check_value_counts_f64(engine, x)


def _last_slot_keys(count: int, slots: int, seed: int) -> np.ndarray:
    """``count`` distinct finite non-zero doubles whose start slot splitmix64(bits) & (s - 1) is s - 1 for every table
    size s <= ``slots`` (their low log2(slots) hash bits are all ones)."""
    rng = np.random.default_rng(seed)
    found, mask = [], np.uint64(slots - 1)
    while sum(f.size for f in found) < count:
        bits = rng.integers(1, 0x7FF0000000000000, 1 << 22, dtype=np.uint64)
        bits |= rng.integers(0, 2, bits.size, dtype=np.uint64) << np.uint64(63)
        found.append(bits[(bn.splitmix64(bits) & mask) == mask])
    bits = np.unique(np.concatenate(found))[:count]
    assert bits.size == count
    return bits.view(np.float64)


def test_value_counts_f64_every_key_starts_at_the_last_slot(engine):
    keys = _last_slot_keys(2048, 16384, 7)
    once = keys.copy()
    assert _table_slots(once.size) == 4096
    _check_value_counts_f64(engine, once)
    # hot and cold keys in the same warps: a few keys many times, most once or twice, shuffled
    rng = np.random.default_rng(8)
    mult = rng.choice([1, 1, 1, 1, 2, 2, 3, 12], keys.size)
    x = np.repeat(keys, mult)
    rng.shuffle(x)
    assert _table_slots(x.size) == 16384 and (mult == 12).sum() > 100
    mask = np.uint64(_table_slots(x.size) - 1)
    assert ((bn.splitmix64(keys.view(np.uint64)) & mask) == mask).all()
    _check_value_counts_f64(engine, x)


def test_value_counts_f64_capacity_contract(engine):
    rng = np.random.default_rng(9)
    x = rng.integers(0, 1000, 20_000).astype(np.float64)
    x[::97] = np.nan
    u, uc = np.unique(x, return_counts=True, equal_nan=True)  # one NaN group
    exp = {(0x7FF8000000000000 if np.isnan(k) else int(k.view(np.uint64))): int(c) for k, c in zip(u, uc)}
    nd_exact = len(exp)
    lib, ctx = engine._lib, engine._ctx

    def call(cap, with_buffers=True):
        keys = np.zeros(max(cap, 1), np.float64)
        counts = np.zeros(max(cap, 1), np.uint64)
        nd = C.c_int64(-1)
        rc = lib.lo_value_counts_f64_host(ctx, x.ctypes.data_as(C.c_void_p), x.size,
                                          keys.ctypes.data_as(C.c_void_p) if with_buffers else None,
                                          counts.ctypes.data_as(C.c_void_p) if with_buffers else None, cap, C.byref(nd), None)
        return rc, nd.value, keys[:cap], counts[:cap]

    rc, nd, keys, counts = call(nd_exact - 1)
    assert rc == N.LO_ERR_INVALID and nd == nd_exact
    assert b"do not fit" in lib.lo_last_error()
    part = dict(zip(keys.view(np.uint64).tolist(), counts.tolist()))
    assert len(part) == nd_exact - 1 and all(exp[k] == c for k, c in part.items())   # what was written is exact
    rc, nd, keys, counts = call(nd_exact)
    assert rc == N.LO_OK and nd == nd_exact
    assert dict(zip(keys.view(np.uint64).tolist(), counts.tolist())) == exp
    rc, nd, _, _ = call(0, with_buffers=False)
    assert rc == N.LO_ERR_INVALID and nd == nd_exact


# ---- text $group --------------------------------------------------------------------------------------------------
def _check_value_counts_str(engine, cells):
    rep, counts = engine.value_counts_str_host(cells)
    got = {cells[int(r)]: int(c) for r, c in zip(rep, counts)}     # each representative row holds its group's bytes
    assert len(got) == len(rep)
    assert got == dict(Counter(cells))


def _collision_columns():
    fx = json.loads((GOLD / "hash_collisions.json").read_text())
    assert fx["table_slots"] == _table_slots(512)
    pairs = [(p["a"], p["b"]) for p in fx["pairs"]]
    cols = []
    # the two cells of a pair in the same warp, either one first
    cols.append([c for a, b in pairs for c in (a, b)])
    cols.append([c for a, b in pairs for c in (b, a, b)])
    # in different warps, with different multiplicities, padded with ordinary cells
    col = []
    for i, (a, b) in enumerate(pairs):
        col += [a] * (i + 1) + [f"pad{i}-{j}" for j in range(40)] + [b] * (2 * i + 3)
    cols.append(col)
    # every member of every pair many times, interleaved across all the warps of a 512-cell column
    rng = np.random.default_rng(2)
    flat = [c for p in pairs for c in p]
    cols.append([flat[i] for i in rng.integers(0, len(flat), 512)])
    return cols


def test_value_counts_str_tag_and_slot_collisions(engine):
    for cells in _collision_columns():
        assert len(cells) <= 512
        _check_value_counts_str(engine, cells)


EDGE_CELLS = [b"", b"\x00", b"\x00\x00", b"ab", b"ab\x00", b"\x00ab", b"\xff", b"\xff\xff", b"\xffab", b"a",
              b"x" * 100_000 + b"\x00", b"x" * 100_000 + b"\x01"]


@pytest.mark.parametrize("n", [1, 31, 32, 33])
def test_value_counts_str_byte_edge_cells(engine, n):
    rng = np.random.default_rng(100 + n)
    cells = [EDGE_CELLS[i] for i in rng.integers(0, len(EDGE_CELLS), n)]
    if n == 1:
        cells = [EDGE_CELLS[-1]]
    elif n == 33:
        cells[-2:] = EDGE_CELLS[-2:]                           # the two long cells that differ in their last byte
    _check_value_counts_str(engine, cells)


def test_value_counts_str_row_limit_is_checked_before_the_offsets(engine):
    lib = engine._lib
    offsets = np.zeros(2, np.int64)                            # far fewer than n + 1 entries: must not be read
    chars = np.zeros(1, np.uint8)
    rows, counts, nd = np.zeros(1, np.int64), np.zeros(1, np.uint64), C.c_int64(-1)
    rc = lib.lo_value_counts_str_host(engine._ctx, chars.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p),
                                      2 ** 31, rows.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), 1,
                                      C.byref(nd), None)
    assert rc == N.LO_ERR_INVALID and b"2^31-1 rows" in lib.lo_last_error()


def test_value_counts_str_packed_on_a_sliced_arrow_column(engine):
    import pyarrow as pa
    from learningorchestra_b200.column_store import TextColumn
    rng = np.random.default_rng(6)
    words = ["", "a", "ab", "male", "female", "é", "x" * 70] + [f"w{i}" for i in range(300)]
    full = pa.array([words[i] for i in rng.integers(0, len(words), 5000)], type=pa.large_string())
    arr = full.slice(1234, 2500)
    assert arr.offset == 1234
    chars, offsets, nulls = TextColumn(arr).packed()
    assert nulls is None and offsets[0] == 0
    rep, counts = engine.value_counts_str_packed(chars, offsets)
    cells = arr.to_pylist()
    got = {cells[int(r)]: int(c) for r, c in zip(rep, counts)}
    assert len(got) == len(rep) and got == dict(Counter(cells))


# ---- range pre-pass -----------------------------------------------------------------------------------------------
def _check_minmax(got, cols, col_idx):
    mins, maxs, cnt = got
    for j, c in enumerate(col_idx):
        mn, mx, nf = _ref_minmax(cols[c])
        assert int(cnt[j]) == nf, (j, c)
        assert mins[j].view(np.uint32) == np.float32(mn).view(np.uint32), (j, c, mins[j], mn)
        assert maxs[j].view(np.uint32) == np.float32(mx).view(np.uint32), (j, c, maxs[j], mx)


def test_minmax_prepass_edges_on_every_route(engine):
    import torch
    from learningorchestra_b200.sharding import ShardedEngine
    n = 3_000_017
    cols = _prepass_columns(n)
    col_idx = [8, 0, 3, 3, 5, 1, 7, 2, 6, 4, 9, 0, 4]
    assert sorted(set(col_idx)) == list(range(len(cols)))
    # the expectations this test pins, beyond agreeing with the reference
    assert _ref_minmax(cols[2])[:2] == (np.float32(F32_MAX), np.float32(F32_MAX))
    assert np.float32(_ref_minmax(cols[4])[0]).view(np.uint32) == 0x80000000
    _check_minmax(engine.minmax_cast_host([cols[c] for c in col_idx]), cols, col_idx)
    t = engine.table_from_numpy(cols)
    try:
        _check_minmax(engine.minmax_cast(t, col_idx), cols, col_idx)
    finally:
        t.free()
    with ShardedEngine.local(list(range(torch.cuda.device_count()))) as eng:
        st = eng.table_from_numpy(cols)
        try:
            _check_minmax(eng.minmax_cast(st, col_idx), cols, col_idx)
        finally:
            st.free()


# ---- the *_host pipeline over more chunks than staging slots --------------------------------------------------------
TILE_ROWS = 61440            # lo::kTileRows: chunk granularity of the f64 pipelines
U8_CHUNK_ROWS = 61440        # lo::kU8HostChunkRows
U32_TILE_ROWS = 1 << 16      # lo_value_counts_u32_host
SLOTS = 3


def _nchunks(nrows, k, elem_bytes, tile_rows, chunk_mb=1):
    """Chunks of a *_host call (loexec.cu, chunk_rows_for): about chunk_mb MiB of input each, whole tiles."""
    target = (chunk_mb << 20) // (k * elem_bytes)
    rows = max(tile_rows, (target // tile_rows) * tile_rows)
    rows = min(rows, -(-nrows // tile_rows) * tile_rows)
    return -(-nrows // rows), rows


def _host_cols(engine, arrays, pinned):
    if not pinned:
        return [np.ascontiguousarray(a) for a in arrays]
    out = []
    for a in arrays:
        p = engine.pinned_empty(a.shape, a.dtype)
        p[:] = a
        out.append(p)
    return out


def _rows_for(k, elem_bytes, tile_rows, chunks=6, ragged=12345):
    _, rows = _nchunks(1 << 40, k, elem_bytes, tile_rows)
    n = rows * (chunks - 1) + ragged
    nch, _ = _nchunks(n, k, elem_bytes, tile_rows)
    assert nch == chunks and nch > SLOTS + 1 and n % rows != 0
    return n, nch


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
def test_host_pipeline_many_chunks(engine, monkeypatch, pinned):
    monkeypatch.setenv("LOEXEC_CHUNK_MB", "1")
    rng = np.random.default_rng(41 + pinned)

    # project + cast + histogram, with outputs and histogram only
    k = 3
    n, nch = _rows_for(k, 8, TILE_ROWS)
    table = bn.synth_table_f64(1, 5150 + pinned, k, 0, n)
    cols = _host_cols(engine, list(table), pinned)
    lo = np.array([-1000.0, -500.0, -1000.0], np.float32)
    hi = np.array([1000.0, 500.0, 999.5], np.float32)
    exp_out, exp_counts = bn.project_cast_hist(table, range(k), 100, lo, hi)
    outs = _host_cols(engine, [np.zeros(n, np.float32) for _ in range(k)], pinned)
    counts, timing = engine.project_cast_hist_host(cols, 100, lo, hi, out=outs)
    np.testing.assert_array_equal(counts, exp_counts)
    for o, e in zip(outs, exp_out):
        np.testing.assert_array_equal(o.view(np.uint32), e.view(np.uint32))
    assert timing["h2d_bytes"] == n * 8 * k and timing["launches"] >= nch
    counts, timing = engine.project_cast_hist_host(cols, 100, lo, hi)
    np.testing.assert_array_equal(counts, exp_counts)
    assert timing["h2d_bytes"] == n * 8 * k and timing["launches"] >= nch

    # byte histogram
    k = 4
    n, nch = _rows_for(k, 1, U8_CHUNK_ROWS, ragged=777)
    u8 = [rng.integers(0, 256, n, dtype=np.uint8) for _ in range(k)]
    u8[1][::3] = 7
    counts, timing = engine.hist_u8_cols_host(_host_cols(engine, u8, pinned))
    np.testing.assert_array_equal(counts, np.stack([np.bincount(c, minlength=256) for c in u8]).astype(np.uint64))
    assert timing["h2d_bytes"] == n * k and timing["launches"] >= nch

    # dictionary-code counts
    n, _ = _rows_for(1, 4, U32_TILE_ROWS, ragged=999)
    codes = rng.integers(0, 5000, n).astype(np.uint32)
    got = engine.value_counts_u32_host(_host_cols(engine, [codes], pinned)[0], 5000)
    np.testing.assert_array_equal(got, np.bincount(codes, minlength=5000))

    # range pre-pass
    idx = [2, 4, 7, 8, 9]            # FLT_MAX, +-0, one finite value at the last / the middle row, normal values
    n, _ = _rows_for(len(idx), 8, TILE_ROWS, ragged=101)
    pre = _prepass_columns(n)
    _check_minmax(engine.minmax_cast_host(_host_cols(engine, [pre[c] for c in idx], pinned)), pre, idx)


def test_host_calls_on_separately_allocated_pinned_columns(engine):
    """Page-locked columns from separate ``pinned_empty`` calls can sit at a constant stride, which the pipeline's
    one-2-D-copy-per-run path must not treat as one allocation; a failed attempt must not leak into the next call."""
    n, k = 100_003, 4
    table = bn.synth_table_f64(1, 77, k, 0, n)
    cols = _host_cols(engine, list(table), True)
    outs = _host_cols(engine, [np.zeros(n, np.float32) for _ in range(k)], True)
    exp_out, exp_counts = bn.project_cast_hist(table, range(k), 64, [-1000.0] * k, [1000.0] * k)
    counts, timing = engine.project_cast_hist_host(cols, 64, -1000.0, 1000.0, out=outs)
    np.testing.assert_array_equal(counts, exp_counts)
    for o, e in zip(outs, exp_out):
        np.testing.assert_array_equal(o.view(np.uint32), e.view(np.uint32))
    u8 = _host_cols(engine, [np.arange(n, dtype=np.uint64).astype(np.uint8) ^ np.uint8(j) for j in range(k)], True)
    counts, _ = engine.hist_u8_cols_host(u8)
    np.testing.assert_array_equal(counts, np.stack([np.bincount(c, minlength=256) for c in u8]).astype(np.uint64))
    vals, st = engine.parse_number_host(["1.5", "x", "7"])          # launches a kernel and checks cudaGetLastError
    assert st.tolist() == [N.LO_NUM_FLOAT, N.LO_NUM_INVALID, N.LO_NUM_INTEGER] and vals[0] == 1.5


# ---- binned histograms without range: auto_range end to end -------------------------------------------------------
AUTO_RANGE_CASES = {
    "subnormal_pair": ([0.0, 1e-45], 10),
    "subnormal_pair_256": ([0.0, 1e-44], 256),
    "flt_max": ([F32_MAX], 10),
    "minus_flt_max": ([-F32_MAX], 10),
}


def _column_values(vals, n=997):
    x = np.array(vals, np.float64)[np.arange(n) % len(vals)]
    x[::5] = np.nan                                            # nulls / NaNs take no part
    return x


def _databases(name, x):
    from learningorchestra_b200.column_store import ColumnarDatabase, NumberColumn
    docs = utils.Database()
    docs.insert_one_in_file(name, rsem.dataset_metadata(name, ["x"]))
    docs.insert_many_in_file(name, [{"_id": i + 1, "x": None if np.isnan(v) else float(v)} for i, v in enumerate(x)])
    cdb = ColumnarDatabase()
    cdb.ingest_columns(name, {"x": NumberColumn(x, ~np.isnan(x))})
    return [("documents", docs), ("columnar", cdb)]


@pytest.mark.parametrize("case", sorted(AUTO_RANGE_CASES))
def test_binned_histogram_without_range_on_degenerate_columns(engine, case):
    vals, nbins = AUTO_RANGE_CASES[case]
    x = _column_values(vals)
    f = bn.cast_f64_f32(x)
    fin = f[np.isfinite(f)]
    lo, hi = bn.auto_range([fin.min()], [fin.max()], [fin.size], nbins)
    engine.resident.clear()
    try:
        for kind, db in _databases("d", x):
            c = Client(server.create_app(db, engine, synchronous=True))
            r = c.post("/histograms", json={"inputDatasetName": "d", "outputDatasetName": "h", "names": ["x"], "bins": nbins})
            assert r.status_code == 201
            meta = db.find_one("h", {"_id": 0})
            assert meta["finished"] is True, (kind, meta)
            doc = [d for d in db.find("h", {}) if d["_id"] != 0][0]["x"]
            assert doc["range"] == [float(lo[0]), float(hi[0])], kind
            assert doc["counts"] == bn.hist_f32(f, lo[0], hi[0], nbins).tolist(), kind
            assert sum(doc["counts"]) == fin.size
    finally:
        engine.resident.clear()


def test_binned_histogram_without_range_fails_when_the_span_overflows_fp32(engine):
    """{-3e38, 3e38}: hi - lo overflows fp32, no finite fp32 range of that width exists, and the job fails with the
    library's message instead of counting with a range it made up."""
    x = _column_values([-3e38, 0.0, 3e38])
    engine.resident.clear()
    try:
        for kind, db in _databases("d", x):
            c = Client(server.create_app(db, engine, synchronous=True))
            r = c.post("/histograms", json={"inputDatasetName": "d", "outputDatasetName": "h", "names": ["x"], "bins": 10})
            assert r.status_code == 201
            meta = db.find_one("h", {"_id": 0})
            assert meta["finished"] is False, kind
            assert "histogram range of column 0 is not usable" in meta["exception"], (kind, meta)
    finally:
        engine.resident.clear()
