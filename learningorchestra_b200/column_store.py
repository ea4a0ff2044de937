"""``ColumnarDatabase`` — the reference's ``Database`` wrapper API over a store that keeps DATA ROWS as columns.

The reference's table is one Mongo document per CSV row, every value a ``str``, ``_id`` = 1-based row number, plus the
metadata document ``_id: 0`` (``database_api_image/database.py:110-151``).  Each of the three hot-path services
scans those documents again for every field.  Here the rows of a dataset live as one array per field —

* :class:`TextColumn`   — Arrow ``large_string`` (chars + int64 offsets + validity): exactly the packed layout the GPU
  parser (``lo_parse_number_host``) and the byte-wise group-by (``lo_value_counts_str_host``) read, so a column goes to
  the device without touching its cells;
* :class:`NumberColumn` — float64 values + valid mask + "stored as int" mask (what ``float(x)`` / ``int(v)`` of
  ``data_type_update.py:40-43`` leave behind);
* :class:`ObjectColumn` — anything else, cell by cell —

while everything that is not a data row (the metadata document, histogram result documents) stays a plain document.
The wrapper methods of :class:`~learningorchestra_b200.utils.Database` (``find``, ``find_one``, ``find_in_file``,
``insert_one_in_file`` ...) behave exactly as before — documents are materialised on demand, page by page for the REST
reader — and the executors use the column accessors when they find them (``has_columns`` / ``column`` / ``set_column``).
A write that addresses individual rows (``update_one`` / ``update_by_id`` / ``insert_one_in_file`` of a data row)
turns the collection back into documents first, so nothing depends on the fast path for correctness.

:meth:`ColumnarDatabase.ingest_csv` is the producer of the format (``Csv.__download_row`` / ``__treat_row`` /
``__save_row``): header names sanitised with ``re.sub(r"\\W+", "", name)``, every cell a string, ``_id`` from 1,
metadata document with ``fields`` and ``finished: True``.
"""
from __future__ import annotations

import math
import re
from collections import OrderedDict

import numpy as np

from .utils import DOCUMENT_ID_NAME, METADATA_DOCUMENT_ID, Database, _matches, _now, record_exception


class NumberColumn:
    """values: float64 (NaN where null); valid: bool; is_int: bool (the document holds a Python ``int``)."""
    kind = "number"

    def __init__(self, values, valid=None, is_int=None):
        self.values = np.ascontiguousarray(values, dtype=np.float64)
        n = self.values.shape[0]
        self.valid = np.ones(n, dtype=bool) if valid is None else np.ascontiguousarray(valid, dtype=bool)
        self.is_int = np.zeros(n, dtype=bool) if is_int is None else np.ascontiguousarray(is_int, dtype=bool)

    def __len__(self):
        return self.values.shape[0]

    def to_pylist(self, start=0, stop=None):
        stop = len(self) if stop is None else stop
        v, ok, ii = self.values[start:stop].tolist(), self.valid[start:stop].tolist(), self.is_int[start:stop].tolist()
        return [None if not o else (int(x) if i else x) for x, o, i in zip(v, ok, ii)]

    def take(self, index):
        return NumberColumn(self.values[index], self.valid[index], self.is_int[index])

    @property
    def integers_collapsed(self) -> bool:
        """Every finite integral value is stored as ``int`` (true after the reference's "number" cast)."""
        v = self.values[self.valid]
        integral = np.isfinite(v) & (v == np.floor(v))
        return bool(np.array_equal(integral, self.is_int[self.valid]))


def large_text(cells):
    """One single-chunk Arrow ``large_string`` array of ``cells``: a list of ``str`` / None, a ``ChunkedArray`` or any
    Arrow string array.  A ``large_string`` array comes back as it is, same buffers."""
    import pyarrow as pa
    arr = cells if isinstance(cells, (pa.Array, pa.ChunkedArray)) else pa.array(cells, type=pa.large_string())
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
    return arr if pa.types.is_large_string(arr.type) else arr.cast(pa.large_string())


class TextColumn:
    """arr: ``pyarrow.LargeStringArray`` (null = ``None``)."""
    kind = "text"

    def __init__(self, arr):
        self.arr = large_text(arr)

    def __len__(self):
        return len(self.arr)

    def to_pylist(self, start=0, stop=None):
        stop = len(self) if stop is None else stop
        return self.arr.slice(start, stop - start).to_pylist()

    def take(self, index):
        import pyarrow as pa
        return TextColumn(self.arr.take(pa.array(np.asarray(index, dtype=np.int64))))

    def packed(self):
        """(chars uint8, offsets int64[n+1] starting at 0, null mask or None): the column's
        :func:`columnar.text_buffers`, rebased by :func:`columnar.zero_based`, and its nulls as a bool array."""
        from .columnar import text_buffers, zero_based
        nulls = np.asarray(self.arr.is_null().to_numpy(zero_copy_only=False), dtype=bool) if self.arr.null_count else None
        return (*zero_based(*text_buffers(self.arr)[:2]), nulls)


class ObjectColumn:
    kind = "object"

    def __init__(self, values):
        self.values = list(values)

    def __len__(self):
        return len(self.values)

    def to_pylist(self, start=0, stop=None):
        return self.values[start:stop]

    def take(self, index):
        return ObjectColumn([self.values[int(i)] for i in index])


class ProbabilityColumn:
    """A prediction dataset's ``probability``: the n x C float64 matrix of a classifier's class probabilities.  A row's
    cell is the list of its C floats, as the reference stores ``probability.toArray().tolist()``; the lists are built
    only for the rows that are read.  Its ``kind`` is ``"object"``, so readers treat it like any column of list cells."""
    kind = "object"

    def __init__(self, matrix):
        self.matrix = np.ascontiguousarray(matrix, dtype=np.float64)
        if self.matrix.ndim != 2:
            raise ValueError(f"a probability column is an n x C matrix, not of shape {self.matrix.shape}")

    def __len__(self):
        return self.matrix.shape[0]

    def to_pylist(self, start=0, stop=None):
        return self.matrix[start:stop].tolist()

    def take(self, index):
        return ProbabilityColumn(self.matrix[np.asarray(index, dtype=np.int64)])


def column_from_values(values):
    """Classify a list of document values: all ``str`` / None -> TextColumn; all int / float / None (no bool, ints that
    float64 holds exactly) -> NumberColumn; anything else -> ObjectColumn."""
    import pyarrow as pa
    try:
        arr = pa.array(values)
    except Exception:          # mixed types
        return ObjectColumn(values)
    t = arr.type
    if pa.types.is_string(t) or pa.types.is_large_string(t):
        return TextColumn(arr)
    if pa.types.is_null(t):
        return NumberColumn(np.full(len(values), math.nan), np.zeros(len(values), dtype=bool))
    if pa.types.is_integer(t) or pa.types.is_floating(t):
        import pyarrow.compute as pc
        if pa.types.is_integer(t):
            mm = pc.min_max(arr)
            lo, hi = mm["min"].as_py(), mm["max"].as_py()
            if lo is not None and (abs(lo) > 2 ** 53 or abs(hi) > 2 ** 53):
                return ObjectColumn(values)
        valid = ~np.asarray(arr.is_null().to_numpy(zero_copy_only=False), dtype=bool)
        vals = np.asarray(pc.cast(arr, pa.float64()).fill_null(math.nan).to_numpy(zero_copy_only=False), dtype=np.float64)
        if pa.types.is_integer(t):
            return NumberColumn(vals, valid, valid.copy())
        # a float-typed Arrow array may have swallowed Python ints (pa.array([1, 2.5]) -> double): recover who was an int
        is_int = np.fromiter((isinstance(v, int) for v in values), dtype=bool, count=len(values))
        return NumberColumn(vals, valid, is_int)
    return ObjectColumn(values)


def _tokenize_pyarrow(source):
    """(header names, Arrow columns, rows, None) by pyarrow.csv; every column read as text, a malformed body raises."""
    import pyarrow as pa
    import pyarrow.csv as pacsv
    # the header first: every column is read as text
    read = pacsv.ReadOptions(autogenerate_column_names=False)
    head = pacsv.open_csv(source, read_options=read, parse_options=pacsv.ParseOptions(newlines_in_values=True)) \
        if isinstance(source, str) else None
    if head is not None:
        raw_names = list(head.schema.names)
        head.close()
    else:
        pos = source.tell()
        first = source.readline()
        source.seek(pos)
        import csv as _csv
        raw_names = next(_csv.reader([first.decode("utf-8") if isinstance(first, bytes) else first]))
    conv = pacsv.ConvertOptions(column_types={n: pa.large_string() for n in raw_names}, strings_can_be_null=False,
                                quoted_strings_can_be_null=False)
    table = pacsv.read_csv(source, read_options=read, convert_options=conv,
                           parse_options=pacsv.ParseOptions(newlines_in_values=True))
    return list(table.schema.names), list(table.columns), table.num_rows, None


def _csv_failure(kind, record, pos):
    """The exception the reference's reader raises for a device reader failure (LO_CSV_*), for the metadata."""
    import csv as _csv

    from . import _native as N
    at = f" (record {record}, byte {pos})"
    if kind == N.LO_CSV_SHORT_ROW:
        return IndexError(f"list index out of range: record {record} has fewer fields than the header")
    if kind == N.LO_CSV_FIELD_LIMIT:
        return _csv.Error(f"field larger than field limit (131072){at}")
    if kind == N.LO_CSV_NUL:
        return _csv.Error(f"line contains NUL{at}")
    if kind == N.LO_CSV_BAD_UTF8:
        return UnicodeDecodeError("utf-8", b"", 0, 0, f"invalid UTF-8 in the line starting at byte {pos} (record {record})")
    if kind == N.LO_CSV_EMPTY:
        return StopIteration("the body has no header")
    return ValueError(f"a line ends inside a UTF-8 sequence{at}: not supported")


def _tokenize_device(read_csv, source):
    """(header cells or None, Arrow columns, rows, failure exception or None) by the engine's GPU reader; the columns
    are zero-copy views of one shared chars buffer."""
    import pyarrow as pa
    if isinstance(source, str):
        body = np.fromfile(source, dtype=np.uint8)
    else:
        data = source.read()
        body = np.frombuffer(data.encode("utf-8") if isinstance(data, str) else data, dtype=np.uint8)
    header, n, chars, offsets, failure = read_csv(body)
    exc = None if failure is None else _csv_failure(*failure)
    if header is None:
        return None, [], 0, exc
    data = pa.py_buffer(chars)
    columns = [pa.LargeStringArray.from_buffers(n, pa.py_buffer(offsets[c, 1:]), data) for c in range(len(header))]
    return header, columns, n, exc


def _tokenize_stream(read_stream, source):
    """(header cells or None, Arrow columns, rows, failure exception or None) by the engine's GPU reader, the source
    streamed from its path or file object in windows."""
    header, n, columns, failure = read_stream(source)
    exc = None if failure is None else _csv_failure(*failure)
    if header is None:
        return None, [], 0, exc
    return header, columns, n, exc


class _Table:
    def __init__(self, ids, columns):
        self.ids = np.ascontiguousarray(ids, dtype=np.int64)
        self.columns: "OrderedDict[str, object]" = OrderedDict(columns)
        self._pos = None

    @property
    def nrows(self):
        return self.ids.shape[0]

    def row(self, i: int) -> dict:
        d = {name: col.to_pylist(i, i + 1)[0] for name, col in self.columns.items()}
        d[DOCUMENT_ID_NAME] = int(self.ids[i])
        return d

    def rows(self, start=0, stop=None) -> list:
        stop = self.nrows if stop is None else min(stop, self.nrows)
        if stop <= start:
            return []
        names = list(self.columns)
        cols = [self.columns[n].to_pylist(start, stop) for n in names]
        ids = self.ids[start:stop].tolist()
        out = []
        for r in range(stop - start):
            d = {n: c[r] for n, c in zip(names, cols)}
            d[DOCUMENT_ID_NAME] = ids[r]
            out.append(d)
        return out

    def position(self, row_id):
        if self._pos is None:
            if self.nrows and np.array_equal(self.ids, np.arange(1, self.nrows + 1)):
                self._pos = "dense"
            else:
                self._pos = {int(v): i for i, v in enumerate(self.ids.tolist())}
        if self._pos == "dense":
            return int(row_id) - 1 if isinstance(row_id, int) and 1 <= row_id <= self.nrows else None
        return self._pos.get(row_id)


class ColumnarDatabase(Database):
    """Drop-in for :class:`~learningorchestra_b200.utils.Database` whose data rows may live as columns."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._tables: dict = {}

    # ---- column accessors (what the executors look for) ---------------------------------------------------
    def has_columns(self, filename) -> bool:
        with self._lock:
            return filename in self._tables

    def nrows(self, filename) -> int:
        with self._lock:
            t = self._tables.get(filename)
            return t.nrows if t is not None else 0

    def row_ids(self, filename):
        with self._lock:
            return self._tables[filename].ids

    def column_names(self, filename):
        with self._lock:
            return list(self._tables[filename].columns)

    def column(self, filename, field):
        """The field's column, or None when no data row has the field."""
        with self._lock:
            return self._tables[filename].columns.get(field)

    def set_column(self, filename, field, column) -> None:
        with self._lock:
            t = self._tables[filename]
            if len(column) != t.nrows:
                raise ValueError(f"column of {len(column)} rows for a table of {t.nrows}")
            t.columns[field] = column
            self._touch(filename)

    def create_table(self, filename, ids, columns) -> None:
        """Data rows of ``filename`` := the given columns (replaces any rows the collection had)."""
        with self._lock:
            docs = self._collections.setdefault(filename, [])
            docs[:] = [d for d in docs if d.get(DOCUMENT_ID_NAME) == METADATA_DOCUMENT_ID]
            self._tables[filename] = _Table(ids, columns)
            self._touch(filename)

    def other_documents(self, filename):
        """Documents of the collection that are not columnar data rows (the metadata document, result documents)."""
        with self._lock:
            return [dict(d) for d in self._collections.get(filename, [])]

    def to_documents(self, filename) -> None:
        """Turn the columnar rows back into plain documents (row-addressed writes need this)."""
        with self._lock:
            t = self._tables.pop(filename, None)
            if t is not None:
                self._collections.setdefault(filename, []).extend(t.rows())

    # ---- the producer of the format: database_api_image/database.py:110-151 -------------------------------
    def ingest_csv(self, filename, source, url=None, engine=None):
        """``POST /files``'s work: ``source`` is a path or a file object of CSV text.  Header sanitised with
        ``re.sub(r"\\W+", "", name)`` (``database.py:118-119``); every cell a string (``:124-137``); ``_id`` from 1;
        metadata document as ``database_api_image/utils.py:50-63`` writes it, ``finished`` flipped to True and
        ``fields`` = the sanitised header at the end (``database.py:139-151``).

        With an engine that has ``read_csv_host`` the body is tokenised on the GPU with the reference's own
        ``csv.reader`` rules: a body the reference fails on keeps the data rows before the failing record, ``finished``
        stays False and the metadata's ``exception`` says why (a failing header stores no rows).  An engine with
        ``read_csv_stream`` streams the source through the reader in windows, so the body's size is bounded by
        neither device nor host memory.  Without an engine, pyarrow tokenises it and a malformed body raises."""
        self.insert_one_in_file(filename, {"datasetName": filename, "url": url, "timeCreated": _now(), "_id": 0,
                                           "finished": False, "type": "dataset/csv"})
        read_stream = getattr(engine, "read_csv_stream", None)
        read_csv = getattr(engine, "read_csv_host", None)
        if read_stream is not None:
            raw_names, columns, n, failure = _tokenize_stream(read_stream, source)
        elif read_csv is not None:
            raw_names, columns, n, failure = _tokenize_device(read_csv, source)
        else:
            raw_names, columns, n, failure = _tokenize_pyarrow(source)
        cols = OrderedDict()
        if raw_names is not None:
            names = [re.sub(r"\W+", "", name) for name in raw_names]
            for name, arr in zip(names, columns):
                cols[name] = TextColumn(arr)           # a repeated sanitised name keeps the LAST column, as dict(zip()) does
            self.create_table(filename, np.arange(1, n + 1, dtype=np.int64), cols)
        if failure is not None:
            record_exception(self, filename, failure)
            return n
        self.update_one(filename, {"finished": True, "fields": list(cols)}, {"_id": 0})
        return n

    def ingest_columns(self, filename, columns: dict, fields=None, url=None):
        """Register ready-made columns (numpy arrays / Arrow string arrays / Column objects) as a finished dataset."""
        cols = OrderedDict()
        n = None
        for name, c in columns.items():
            if not hasattr(c, "kind"):
                import pyarrow as pa
                if isinstance(c, (pa.Array, pa.ChunkedArray)):
                    c = TextColumn(c)
                else:
                    a = np.asarray(c)
                    c = NumberColumn(a.astype(np.float64), ~np.isnan(a.astype(np.float64)), np.issubdtype(a.dtype, np.integer) & np.ones(a.shape[0], bool))
            cols[name] = c
            n = len(c) if n is None else n
            if len(c) != n:
                raise ValueError("columns of different lengths")
        self.insert_one_in_file(filename, {"datasetName": filename, "url": url, "timeCreated": _now(), "_id": 0,
                                           "finished": True, "type": "dataset/csv", "fields": list(fields or cols)})
        self.create_table(filename, np.arange(1, (n or 0) + 1, dtype=np.int64), cols)
        return n or 0

    # ---- wrapper API: reads -----------------------------------------------------------------------------------
    def find(self, filename, query):
        with self._lock:
            docs = super().find(filename, query)
            t = self._tables.get(filename)
            if t is None:
                return docs
            if set(query) == {DOCUMENT_ID_NAME} and not isinstance(query[DOCUMENT_ID_NAME], dict):
                p = t.position(query[DOCUMENT_ID_NAME])
                return docs + ([t.row(p)] if p is not None else [])
            rows = t.rows()
            return docs + (rows if not query else [d for d in rows if _matches(d, query)])

    def find_one(self, filename, query):
        with self._lock:
            d = super().find_one(filename, query)
            if d is not None:
                return d
            t = self._tables.get(filename)
            if t is None:
                return None
            if set(query) == {DOCUMENT_ID_NAME}:
                p = t.position(query[DOCUMENT_ID_NAME])
                return t.row(p) if p is not None else None
            for start in range(0, t.nrows, 65536):
                for row in t.rows(start, start + 65536):
                    if _matches(row, query):
                        return row
        return None

    def find_in_file(self, filename, query, skip=0, limit=10):
        """``database_api_image/utils.py:17-23``: sorted by ``_id``, then skip / limit — only the page is materialised."""
        with self._lock:
            t = self._tables.get(filename)
            if t is None or query or not (t.nrows == 0 or t.position(1) == 0):
                return super().find_in_file(filename, query, skip, limit) if t is None else \
                    sorted(self.find(filename, query), key=lambda d: d[DOCUMENT_ID_NAME])[skip:skip + limit]
            small = sorted(super().find(filename, {}), key=lambda d: d[DOCUMENT_ID_NAME])
            before = [d for d in small if d[DOCUMENT_ID_NAME] < 1]           # the metadata document
            after = [d for d in small if d[DOCUMENT_ID_NAME] > t.nrows]
            out = before[skip:skip + limit]
            room = limit - len(out)
            if room > 0:
                start = max(0, skip - len(before))
                out += t.rows(start, start + room)
                room = limit - len(out)
                if room > 0:
                    out += after[max(0, skip - len(before) - t.nrows):][:room]
            return out

    # ---- wrapper API: writes ----------------------------------------------------------------------------------
    def insert_one_in_file(self, filename, json_object):
        with self._lock:
            if json_object.get(DOCUMENT_ID_NAME) != METADATA_DOCUMENT_ID and filename in self._tables:
                self.to_documents(filename)
            super().insert_one_in_file(filename, json_object)

    def insert_many_in_file(self, filename, json_objects):
        with self._lock:
            if filename in self._tables:
                self.to_documents(filename)
            super().insert_many_in_file(filename, json_objects)

    def update_one(self, filename, new_value, query):
        with self._lock:
            if filename in self._tables and query.get(DOCUMENT_ID_NAME) != METADATA_DOCUMENT_ID:
                self.to_documents(filename)
            super().update_one(filename, new_value, query)

    def update_by_id(self, filename, updates: dict):
        with self._lock:
            if filename in self._tables and updates:
                self.to_documents(filename)
            super().update_by_id(filename, updates)

    def delete_file(self, filename):
        with self._lock:
            self._tables.pop(filename, None)
            super().delete_file(filename)
