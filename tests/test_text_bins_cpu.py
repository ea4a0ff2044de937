"""CPU: the host side of binned / cast requests on TEXT fields — the one ASCII-mapping rule, the zero-copy Arrow buffers
the device parse reads, the shard summary merge, the ABI mirror of the new structs, and the resident-table logic around
the parse (run against a stand-in whose ``parse_number_into`` is CPython's ``float()``, so no device is needed)."""
import ctypes
import re
import subprocess
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest

from learningorchestra_b200 import columnar, utils
from learningorchestra_b200.column_store import ColumnarDatabase, TextColumn, large_text
from learningorchestra_b200.sharding import combine_parse_summaries
from learningorchestra_b200.table_cache import ResidentTables, is_text_field

ROOT = Path(__file__).resolve().parent.parent


def test_number_text_maps_only_non_ascii_cells_and_keeps_buffers():
    arr = pa.array(["1", None, "2.5", ""], type=pa.large_string())
    assert columnar.number_text(arr) is arr
    mapped = columnar.number_text(["１２", None, " 7 ", "٣.٥", "  5\xa0", "x€"])
    assert mapped.to_pylist() == ["12", None, " 7 ", "3.5", "  5 ", "x?"]
    assert columnar.pack_number_cells(["１２", "3"])[0][:3].tobytes() == b"123"


def test_text_buffers_of_a_sliced_array_with_nulls():
    arr = pa.array([None if i % 3 == 0 else str(i) for i in range(40)], type=pa.large_string()).slice(5, 20)
    chars, offsets, validity = columnar.text_buffers(arr)
    assert offsets.shape == (21,) and offsets[0] != 0
    bitmap, bit0 = validity
    assert bit0 == 5
    for i, cell in enumerate(arr.to_pylist()):
        present = (bitmap[(bit0 + i) >> 3] >> ((bit0 + i) & 7)) & 1
        assert bool(present) == (cell is not None)
        if cell is not None:
            assert chars[offsets[i]:offsets[i + 1]].tobytes().decode() == cell
    assert columnar.text_buffers(pa.array(["a"], type=pa.large_string()))[2] is None
    np.testing.assert_array_equal(columnar.number_text_valid(pa.array(["1", None, "", "x"], type=pa.large_string())),
                                  [True, False, False, True])


def _text_inputs():
    cells = [None if i % 5 == 2 else "é" * (i % 3) + str(i) for i in range(40)]
    large = pa.array(cells, type=pa.large_string())
    return {
        "list": cells[:17],
        "large": large,
        "sliced": large.slice(11, 20),
        "sliced_without_nulls": pa.array([c or "" for c in cells], type=pa.large_string()).slice(3, 30),
        "string": pa.array(cells, type=pa.string()).slice(7, 25),
        "chunked": pa.chunked_array([large.slice(0, 9), pa.array(cells[9:], type=pa.large_string())]),
        "one_chunk": pa.chunked_array([large.slice(5, 10)]),
        "empty": pa.array([], type=pa.large_string()),
        "sliced_empty_tail": pa.array(["ab", "", None, ""], type=pa.large_string()).slice(1),
    }


@pytest.mark.parametrize("name", list(_text_inputs()))
def test_every_text_input_reads_as_one_large_string_array(name):
    src = _text_inputs()[name]
    cells = src if isinstance(src, list) else src.to_pylist()
    n = len(cells)
    arr = large_text(src)
    assert isinstance(arr, pa.Array) and pa.types.is_large_string(arr.type) and arr.to_pylist() == cells
    if isinstance(src, pa.Array) and pa.types.is_large_string(src.type):
        assert arr is src
    chars, offsets, validity = columnar.text_buffers(arr)
    assert chars.dtype == np.uint8 and chars.size >= 1 and offsets.dtype == np.int64 and offsets.shape == (n + 1,)
    if n and arr.buffers()[2] is not None:          # views of the Arrow buffers, the slice's offsets as they are
        assert chars.ctypes.data == arr.buffers()[2].address
        assert offsets.ctypes.data == arr.buffers()[1].address + 8 * arr.offset
    cell_bytes = [chars[offsets[i]:offsets[i + 1]].tobytes() for i in range(n)]
    assert [b.decode() for b, c in zip(cell_bytes, cells) if c is not None] == [c for c in cells if c is not None]
    if None in cells:
        bitmap, bit0 = validity
        assert [not (bitmap[(bit0 + i) >> 3] >> ((bit0 + i) & 7)) & 1 for i in range(n)] == [c is None for c in cells]
    else:
        assert validity is None
    zchars, zoffsets = columnar.zero_based(chars, offsets)
    assert zoffsets[0] == 0 and zoffsets.shape == (n + 1,)
    assert [zchars[zoffsets[i]:zoffsets[i + 1]].tobytes() for i in range(n)] == cell_bytes
    pchars, poffsets, nulls = TextColumn(arr).packed()
    np.testing.assert_array_equal(poffsets, zoffsets)
    assert [pchars[poffsets[i]:poffsets[i + 1]].tobytes() for i in range(n)] == cell_bytes
    assert (nulls is None) if None not in cells else nulls.tolist() == [c is None for c in cells]
    present = [c for c in cells if c is not None]
    pchars, poffsets = columnar.pack_cells(present)
    assert poffsets[0] == 0 and [pchars[poffsets[i]:poffsets[i + 1]].tobytes().decode() for i in range(len(present))] == present


def test_shard_summaries_merge_to_the_global_first_row():
    t = {"total_ms": 1.0, "kernel_ms": 0.5, "h2d_bytes": 10.0, "d2h_bytes": 32.0, "launches": 1}
    parts = [{"first_invalid": None, "first_unsupported": 30, "nulls": 2, "integer": True, **t},
             {"first_invalid": 3, "first_unsupported": None, "nulls": 1, "integer": False, **t},
             {"first_invalid": 0, "first_unsupported": 1, "nulls": 0, "integer": True, **t}]
    s = combine_parse_summaries(parts, [0, 64, 96])
    assert (s["first_invalid"], s["first_unsupported"], s["nulls"], s["integer"]) == (67, 30, 3, False)
    assert s["launches"] == 3 and s["h2d_bytes"] == 30.0 and s["kernel_ms"] == 0.5
    s = combine_parse_summaries(parts[:1], [128])
    assert s["first_invalid"] is None and s["first_unsupported"] == 158 and s["integer"] is True


def test_text_field_classification():
    assert is_text_field(["1", None, ""]) and not is_text_field([None, None]) and not is_text_field(["1", 2])


def test_parse_structs_match_the_header(tmp_path):
    from learningorchestra_b200 import _native
    text = (ROOT / "include" / "loexec.h").read_text()
    assert int(re.search(r"#define LO_ABI_VERSION (\d+)", text).group(1)) == _native.LO_ABI_VERSION
    src = tmp_path / "layout.c"
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "loexec.h"', 'int main(void) {']
    for struct, mirror in (("lo_validity", _native.Validity), ("lo_parse_summary", _native.ParseSummary)):
        lines.append(f'    printf("sizeof.{struct} %zu\\n", sizeof({struct}));')
        lines += [f'    printf("{struct}.{f} %zu\\n", offsetof({struct}, {f}));' for f, _ in mirror._fields_]
    src.write_text("\n".join(lines + ["    return 0;", "}"]) + "\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for struct, mirror in (("lo_validity", _native.Validity), ("lo_parse_summary", _native.ParseSummary)):
        assert int(got[f"sizeof.{struct}"]) == ctypes.sizeof(mirror)
        for f, _ in mirror._fields_:
            assert int(got[f"{struct}.{f}"]) == getattr(mirror, f).offset


# ---- the resident-table logic, with float() standing in for the device --------------------------------------------
class _Table:
    def __init__(self, owner, nrows, ncols):
        self.owner, self.nrows, self.ncols = owner, nrows, ncols
        self.data = np.zeros((ncols, nrows))
        self.pitch_bytes = nrows * 8
        owner.live.add(id(self))

    def upload(self, col, values):
        self.data[col] = values

    def to_numpy(self, col):
        return self.data[col].copy()

    def free(self):
        self.owner.live.discard(id(self))


class _FloatEngine:
    """``table`` / ``parse_number_into`` with CPython's float(): the cell semantics the device kernel implements."""

    def __init__(self):
        self.live, self.parses = set(), 0

    def table(self, dtype, nrows, ncols):
        return _Table(self, nrows, ncols)

    def parse_number_into(self, table, col, chars, offsets, nulls=None):
        self.parses += 1
        n = offsets.shape[0] - 1
        out = {"first_invalid": None, "first_unsupported": None, "nulls": 0, "integer": True}
        for i in range(n):
            if isinstance(nulls, tuple):
                null = not (nulls[0][(nulls[1] + i) >> 3] >> ((nulls[1] + i) & 7)) & 1
            else:
                null = nulls is not None and bool(nulls[i])
            cell = chars[offsets[i]:offsets[i + 1]].tobytes().decode()
            if null or cell == "":
                table.data[col, i] = np.nan
                out["nulls"] += 1
                continue
            try:
                v = float(cell)
            except ValueError:
                out["first_invalid"] = i if out["first_invalid"] is None else out["first_invalid"]
                continue
            table.data[col, i] = v
            out["integer"] = out["integer"] and np.isfinite(v) and v.is_integer()
        return out


def _dbs(columns):
    docs = utils.Database()
    docs.insert_one_in_file("d", {"_id": 0, "finished": True, "fields": list(columns)})
    n = len(next(iter(columns.values())))
    docs.insert_many_in_file("d", [{"_id": i + 1, **{f: c[i] for f, c in columns.items()}} for i in range(n)])
    cdb = ColumnarDatabase()
    cdb.ingest_columns("d", {f: (pa.array(c, type=pa.large_string()) if is_text_field(c) else np.array(c, float))
                             for f, c in columns.items()})
    return [("documents", docs), ("columnar", cdb)]


def test_resident_table_parses_text_and_records_kind_and_nulls():
    cols = {"t": ["1", "", None, "１２", "-3"], "u": ["0.5", "2", None, "", "nan"], "x": [1.0, 2.0, 3.0, 4.0, 5.0]}
    for kind, db in _dbs(cols):
        eng = _FloatEngine()
        cache = ResidentTables(eng)
        data = cache.ensure(db, "d", ["t", "u", "x"])
        assert data.kinds[:2] == ["int", "float"] and data.nulls == [2, 2, 0], kind
        got = data.table.to_numpy(data.column["t"])
        np.testing.assert_array_equal(got, [1.0, np.nan, np.nan, 12.0, -3.0])
        cache.release(data)
        again = cache.ensure(db, "d", ["t"])
        assert cache.hits == 1 and eng.parses == 2, kind
        cache.release(again)


def test_bad_cell_frees_the_table_and_caches_nothing():
    cols = {"a": ["1", "2", "zz", "4"], "b": ["1", "x", "3", "y"], "c": ["1", "2", "3", "4"]}
    for kind, db in _dbs(cols):
        eng = _FloatEngine()
        cache = ResidentTables(eng)
        with pytest.raises(ValueError, match=r"could not convert string to float: 'x'"):
            cache.ensure(db, "d", ["c", "b", "a"])            # b comes before a in the request, its first bad row is 1
        with pytest.raises(ValueError, match=r"could not convert string to float: 'zz'"):
            cache.ensure(db, "d", ["a", "b"])
        assert not cache._entries and not eng.live, kind


def test_mixed_document_fields_keep_their_error():
    docs = utils.Database()
    docs.insert_one_in_file("d", {"_id": 0, "finished": True, "fields": ["m"]})
    docs.insert_many_in_file("d", [{"_id": 1, "m": "1"}, {"_id": 2, "m": 2}])
    with pytest.raises(ValueError, match="is not numeric"):
        ResidentTables(_FloatEngine()).ensure(docs, "d", ["m"])
