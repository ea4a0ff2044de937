"""``DataType`` — drop-in for ``data_type_handler_image/data_type_update.py`` (same constructor and
methods, in-place conversion of the input collection, same ``finished`` False -> True protocol).

* ``"number"`` (``data_type_update.py:30-43``): every text cell of the field is parsed ON THE GPU
  (``lo_parse_number_host`` -> ``k_parse_number``: CPython ``float()`` grammar, correctly rounded binary64,
  plus the ``is_integer()`` flag) — the reference does ``float(document[field])`` one document at a time.
  The adapter keeps the reference's branch order around it: ``None`` untouched, ``""`` -> ``None``, the dead
  ``== int / == float`` checks, integer-valued results stored as ``int``; an unparsable cell raises
  ``ValueError`` after the earlier documents were updated, so the collection is left exactly as the
  reference leaves it (``finished: False``).  Unicode digits / whitespace (``"１２"``, ``"٣.٥"``) are mapped to ASCII by
  the packer exactly as ``float(str)`` maps them (:func:`columnar.ascii_number_text`); a cell over 1 MiB fails the job
  loudly (no host ``float()`` fallback).
* ``"string"`` (``data_type_update.py:22-28``): ``str(v)`` / ``None -> ""``.  With an engine that has
  ``format_number_host``, every number of the field is formatted ON THE GPU in one call (``lo_format_number_host`` ->
  ``k_format_number_len`` / ``_write``: ``repr(float)`` with CPython's shortest round-trip digits, ``str(int)`` of
  integral values, ``""`` for None), the parser's inverse.  A number column comes back as the Arrow ``large_string``
  buffers of a new TextColumn; in documents, the cells that are binary64 numbers go to the device and everything else
  (text, bools, ints beyond a double, other objects) keeps ``str()``.  A failing device call fails the job, with no host
  retry.  An engine without the method (``engine=None``) formats with ``str()`` on the host.
* ``"float32"`` (this build's optional extension): the B-semantics cast of SURVEY.md §0 — numeric values
  go through the sm_90a kernel (fp64 -> fp32 round-to-nearest-even) and are stored back widened.
"""
from __future__ import annotations

from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import columnar
from .utils import record_exception


def _is_binary64(cell) -> bool:
    """A float, or an int (not a bool) that a double holds exactly: the cells the device formatter takes."""
    if type(cell) is float:
        return True
    if type(cell) is not int:
        return False
    try:
        return int(float(cell)) == cell
    except OverflowError:
        return False


class DataType:
    METADATA_DOCUMENT_ID = 0
    DOCUMENT_ID_NAME = "_id"
    STRING_TYPE = "string"
    NUMBER_TYPE = "number"
    FLOAT32_TYPE = "float32"

    def __init__(self, database_connector, metadata_handler, engine=None):
        self.database_connector = database_connector
        self.thread_pool = ThreadPoolExecutor()
        self.metadata_handler = metadata_handler
        self.engine = engine
        self.last_job = None

    def field_converter(self, filename, field, field_type):
        if getattr(self.database_connector, "has_columns", lambda _f: False)(filename):
            return self.__convert_column(filename, field, field_type)
        rows = columnar.data_rows(self.database_connector.find(filename, {}))
        failure = None
        if field_type == self.FLOAT32_TYPE:
            changes = self.__gpu_float32(rows, field)
        elif field_type == self.NUMBER_TYPE:
            changes, failure = self.__gpu_number(rows, field)
        elif field_type == self.STRING_TYPE:
            changes = self.__to_text(rows, field)
        else:
            changes = {}                      # unknown type: the reference issues an empty $set
        self.database_connector.update_by_id(filename, changes)
        if failure is not None:
            raise failure

    def __convert_column(self, filename, field, field_type):
        """The same conversions on a collection stored as columns (:mod:`column_store`): the text column's Arrow
        buffers are the parser's input, the result is a new NumberColumn — no per-document round trip at all (the
        reference does one ``update_one`` per document per field, ``data_type_update.py:45``)."""
        from . import _native as N
        from .column_store import NumberColumn, ObjectColumn, TextColumn
        db = self.database_connector
        col = db.column(filename, field)
        if col is None:
            raise KeyError(field)                       # reference: document[field] raises KeyError on the first row
        if col.kind == "object":                       # mixed cells: the per-document definition decides
            db.to_documents(filename)
            return self.field_converter(filename, field, field_type)
        if field_type == self.STRING_TYPE:
            if col.kind == "text":                     # str(v) of a str is itself; None -> ""
                new = TextColumn(col.arr.fill_null("")) if col.arr.null_count else col
            elif getattr(self.engine, "format_number_host", None) is not None:     # str(int) / repr(float) on the GPU
                import pyarrow as pa
                status = np.where(~col.valid, N.LO_NUM_EMPTY, np.where(col.is_int, N.LO_NUM_INTEGER, N.LO_NUM_FLOAT))
                chars, offsets = self.engine.format_number_host(col.values, status.astype(np.uint8))
                new = TextColumn(pa.LargeStringArray.from_buffers(len(col), pa.py_buffer(offsets), pa.py_buffer(chars)))
            else:                                      # no device formatter: str() on the host
                import pyarrow as pa
                new = TextColumn(pa.array(["" if v is None else str(v) for v in col.to_pylist()], type=pa.large_string()))
            db.set_column(filename, field, new)
        elif field_type == self.NUMBER_TYPE:
            if self.engine is None:
                raise RuntimeError("type 'number' parses text on the GPU and needs an Engine (there is no CPU fallback)")
            if col.kind == "number":                   # float(v); is_integer() -> int(v)
                v = col.values
                integral = col.valid & np.isfinite(v) & (v == np.floor(v))
                db.set_column(filename, field, NumberColumn(v, col.valid, integral))
                return
            import pyarrow.compute as pc
            arr = col.arr
            if not pc.all(pc.string_is_ascii(arr.fill_null(""))).as_py():      # Unicode digits / spaces, as float(str)
                import pyarrow as pa
                arr = pa.array([None if c is None else columnar.ascii_number_text(c) for c in arr.to_pylist()], type=pa.large_string())
            chars, offsets, nulls = TextColumn(arr).packed()
            values, status = self.engine.parse_number_packed(chars, offsets)
            bad = np.flatnonzero((status == N.LO_NUM_INVALID) | (status == N.LO_NUM_UNSUPPORTED))
            if nulls is not None:
                bad = bad[~nulls[bad]]
            if bad.size:
                # the reference converts document by document and dies on the first bad cell: earlier rows converted,
                # the rest untouched, finished stays False
                first = int(bad[0])
                cells = col.to_pylist()
                head = NumberColumn(values[:first], (status[:first] <= N.LO_NUM_INTEGER), status[:first] == N.LO_NUM_INTEGER).to_pylist()
                db.set_column(filename, field, ObjectColumn(head + cells[first:]))
                if status[first] == N.LO_NUM_UNSUPPORTED:
                    raise RuntimeError(f"cell of {len(cells[first])} characters exceeds the device parser's 1 MiB limit "
                                       "and there is no CPU fallback")
                raise ValueError(f"could not convert string to float: {cells[first]!r}")
            valid = status <= N.LO_NUM_INTEGER           # "" (and None) -> None
            db.set_column(filename, field, NumberColumn(np.where(valid, values, np.nan), valid, status == N.LO_NUM_INTEGER))
        elif field_type == self.FLOAT32_TYPE:
            if col.kind != "number":
                raise ValueError(f"field {field!r} is not numeric; convert it to 'number' first")
            if self.engine is None:
                raise RuntimeError("type 'float32' needs an Engine (there is no CPU fallback)")
            out = np.empty(len(col), dtype=np.float32)
            self.engine.project_cast_hist_host([np.ascontiguousarray(col.values)], None, out=[out])
            db.set_column(filename, field, NumberColumn(np.where(col.valid, out.astype(np.float64), np.nan), col.valid))
        # unknown type: the reference issues an empty $set

    def __to_text(self, rows, field):
        """``data_type_update.py:22-28``: ``None -> ""``, anything else ``str(v)``; the reference's guard
        ``document[field] == str`` compares a value with the type object and is never true.

        With a device formatter the cells that are binary64 numbers — ``float``, and ``int`` whose value a double
        holds exactly — are formatted on the GPU in one call (``repr(float)`` / ``str(int)``).  Text, ``bool``
        (``str(True)`` is ``"True"``), ints beyond a double and other objects were never numbers the device holds and
        keep ``str()`` on the host."""
        from . import _native as N
        fmt = getattr(self.engine, "format_number_host", None)
        changes, device_ids, values, status = {}, [], [], []
        for row in rows:
            cell = row[field]
            if cell == str:
                continue
            if fmt is not None and _is_binary64(cell):
                device_ids.append(row[self.DOCUMENT_ID_NAME])
                values.append(float(cell))
                status.append(N.LO_NUM_INTEGER if type(cell) is int else N.LO_NUM_FLOAT)
                changes[row[self.DOCUMENT_ID_NAME]] = None          # keeps the document order; filled below
                continue
            changes[row[self.DOCUMENT_ID_NAME]] = {field: "" if cell is None else str(cell)}
        if device_ids:
            chars, offsets = fmt(np.array(values, dtype=np.float64), np.array(status, dtype=np.uint8))
            raw = chars.tobytes()
            for j, doc_id in enumerate(device_ids):
                changes[doc_id] = {field: raw[offsets[j]:offsets[j + 1]].decode("ascii")}
        return changes

    def __gpu_number(self, documents, field):
        """``data_type_update.py:30-43`` with the ``float(str)`` of every text cell done by the GPU parser."""
        if self.engine is None:
            raise RuntimeError("type 'number' parses text on the GPU and needs an Engine (there is no CPU fallback)")
        from . import _native as N
        text_rows = [i for i, d in enumerate(documents) if isinstance(d[field], str) and d[field] != ""]
        parsed, status = self.engine.parse_number_host([documents[i][field] for i in text_rows])
        where = {row: j for j, row in enumerate(text_rows)}
        updates = {}
        for i, document in enumerate(documents):
            value = document[field]
            if value == int or value == float or value is None:       # :32-36 (first two never true)
                continue
            if value == "":
                new = None
            elif i in where:
                j = where[i]
                if status[j] == N.LO_NUM_INVALID:
                    return updates, ValueError(f"could not convert string to float: {value!r}")
                if status[j] == N.LO_NUM_UNSUPPORTED:
                    return updates, RuntimeError(f"cell {value[:40]!r}... ({len(value)} characters) exceeds the device "
                                                 "parser's 1 MiB cell limit and there is no CPU fallback")
                new = float(parsed[j])
                if status[j] == N.LO_NUM_INTEGER:
                    new = int(new)
            else:                                                        # already a number (or bool): no text to parse
                new = float(value)
                if new.is_integer():
                    new = int(new)
            updates[document[self.DOCUMENT_ID_NAME]] = {field: new}
        return updates, None

    def __gpu_float32(self, documents, field):
        if self.engine is None:
            raise RuntimeError("type 'float32' needs an Engine (there is no CPU fallback)")
        packed = columnar.numeric_column([d.get(field) for d in documents])
        if packed is None:
            raise ValueError(f"field {field!r} is not numeric; convert it to 'number' first")
        col, valid, _kind = packed
        out = np.empty(len(documents), dtype=np.float32)
        self.engine.project_cast_hist_host([col], None, out=[out])
        return {d[self.DOCUMENT_ID_NAME]: {field: float(out[i])} for i, d in enumerate(documents) if valid[i]}

    def convert_existent_file(self, filename, fields_dictionary):
        self.metadata_handler.update_finished_flag(filename, False)
        self.last_job = self.thread_pool.submit(self.field_file_converter, filename, fields_dictionary)

    def field_file_converter(self, filename, fields_dictionary):
        try:
            for field in fields_dictionary:
                self.field_converter(filename, field, fields_dictionary[field])
            self.metadata_handler.update_finished_flag(filename, True)
        except BaseException as exc:
            record_exception(self.database_connector, filename, exc)
            raise

    def wait(self, timeout=None):
        if self.last_job is not None:
            self.last_job.result(timeout)
