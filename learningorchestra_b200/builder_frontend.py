"""The builder service's table front-end (``builder_image/builder.py:172-194``), the fourth "next" row of
SURVEY.md §8f: ``load -> filter(_id != 0) -> drop(metadata columns)`` that feeds Spark ML in the reference.

Only the front-end is mirrored (model building itself is out of scope, SURVEY.md §2): the data rows of a
dataset as a **columnar frame** — ``pyarrow.Table`` on the host, or the HBM-resident slabs themselves
(``ResidentDataset``) for a GPU consumer — with the reference's metadata columns removed.  The connector
infers its schema from a sample that contains the metadata document, so its keys show up as all-null
columns on every data row; that is why the reference drops them, and why ``_id`` goes too.
"""
from __future__ import annotations

from . import columnar

METADATA_FIELDS = ["_id", "fields", "datasetName", "finished", "timeCreated", "url", "parentDatasetName", "type"]


def frame_fields(database, filename):
    """Column names of the processed frame: the dataset's fields minus the metadata columns, in stored order."""
    metadata = database.find_one(filename, {"_id": 0}) or {}
    declared = list(metadata.get("fields") or [])
    rows = columnar.data_rows(database.find(filename, {}))
    seen = list(declared)
    for d in rows[:1000]:                        # the connector samples documents to infer the schema
        for key in d:
            if key not in seen:
                seen.append(key)
    return [f for f in seen if f not in METADATA_FIELDS], rows


def file_processor(database, filename, engine=None):
    """``Builder.__file_processor``: data rows without the metadata columns, as a ``pyarrow.Table`` (rows in
    ``_id`` order).  With an ``engine`` the numeric columns are taken from / registered in the HBM-resident copy
    of the dataset, so a GPU consumer can use ``engine.resident.ensure(...)`` on the same slabs without another
    scan; values are identical either way."""
    import numpy as np
    import pyarrow as pa

    fields, rows = frame_fields(database, filename)
    rows.sort(key=lambda d: d["_id"])
    packed = {f: (columnar.numeric_column([d.get(f) for d in rows]) if rows else None) for f in fields}
    numeric = [f for f in fields if packed[f] is not None]
    resident = engine.resident.ensure(database, filename, numeric) if (engine is not None and numeric) else None
    try:
        return _frame(fields, rows, packed, resident)
    finally:
        if resident is not None:
            engine.resident.release(resident)


class DeviceFrame:
    """The processed frame for a GPU consumer: the HBM-resident slabs themselves, no device->host copy.
    ``columns[name]`` is a list of :class:`~learningorchestra_b200.engine.DeviceColumn` (one per shard: one element on a
    single GPU) exposing ``__cuda_array_interface__`` — nulls are NaN in the slab; ``nulls[name]`` counts them.
    A text field (``device_frame(..., text=True)``) is a column of int32 dictionary codes instead, ``kinds[name] ==
    "text"``: -1 for a null row, else the index of its cell in ``dictionaries[name]``, the Arrow array of the distinct
    cells in the order of their first rows.  The frame owns those code tables (they are not cached) and frees them in
    :meth:`release`.  Holds a lease on the resident dataset: call :meth:`release` (or use ``with``) when the consumer is
    done."""

    def __init__(self, cache, data, fields, codes=None):
        self._cache, self._data = cache, data
        self._codes = dict(codes or {})          # text field -> (code table, dictionary)
        self.fields = list(fields)
        self.ids = data.ids
        shards = getattr(data.table, "shards", [data.table])
        self.columns, self.kinds, self.nulls, self.dictionaries = {}, {}, {}, {}
        for f in self.fields:
            if f in self._codes:
                table, dictionary = self._codes[f]
                self.columns[f] = [t.column_view(0, keepalive=self) for t in getattr(table, "shards", [table])]
                self.kinds[f], self.nulls[f], self.dictionaries[f] = "text", data.texts[f].nulls, dictionary
            else:
                self.columns[f] = [t.column_view(data.column[f], keepalive=self) for t in shards]
                self.kinds[f] = data.kinds[data.column[f]]
                self.nulls[f] = data.nulls[data.column[f]]

    def features(self, fields=None, label=None, dtype: str = "float32", handle_invalid: str = "error") -> "Features":
        """The step the reference's modelingCode ends in before ``classifier.fit``: Spark 2.4's
        ``VectorAssembler(inputCols=fields, outputCol="features")`` and its ``label`` column, assembled in HBM on every
        shard's device (``Engine.assemble_rows``).  Row i is ``[value(f, i) for f in fields]``: a number field's slab
        value, a text field's dictionary code, as ``dtype`` ("float32": round-to-nearest-even; "float64": exact).
        ``fields=None``: every field of the frame but ``label``, in frame order.  A cell is invalid when it is NaN (a null
        or a real NaN) or a null text cell (code -1); ``handle_invalid``: "error" raises LoexecError LO_ERR_INVALID naming
        the ``_id`` and field of the lowest one, "skip" drops every row with one in ``fields`` or ``label``, "keep" writes
        NaN.  A field not in the frame raises KeyError before anything runs."""
        from .engine import InvalidCellError, assemble_args
        from .sharding import ShardedEngine
        assemble_args(handle_invalid, dtype)
        fields = [f for f in self.fields if f != label] if fields is None else list(fields)
        for f in fields + ([label] if label is not None else []):
            if f not in self.columns:
                raise KeyError(f)
        if not fields:
            raise ValueError("features needs at least one field")
        if self._data is None:
            raise ValueError("the frame has been released")
        engine = self._cache.engine
        try:
            parts = engine.assemble_rows([self._source(f) for f in fields],
                                         self._source(label) if label is not None else None, dtype, handle_invalid)
        except InvalidCellError as e:
            raise named_cell(e, fields, label, self.ids, "features", ("is null or NaN (handle_invalid='error')",) * 2) from None
        return Features(self, parts if isinstance(engine, ShardedEngine) else [parts], fields, label, dtype)

    def _source(self, f):
        """(table, column) of field f as ``assemble_rows`` reads it: its code table, or the dataset's slab table."""
        if f in self._codes:
            return self._codes[f][0], 0
        return self._data.table, self._data.column[f]

    def release(self):
        codes, self._codes = self._codes, {}
        for table, _dictionary in codes.values():
            table.free()
        if self._data is not None:
            self._cache.release(self._data)
            self._data = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.release()


def named_cell(e, fields, label, ids, call: str, reasons: tuple[str, str]):
    """A refused cell ``e`` (an :class:`~engine.InvalidCellError` whose row indexes ``ids`` and whose position indexes
    ``fields``, ``len(fields)`` the label) restated for the user: "<call>: field F of the row with _id I <reason>",
    ``reasons[0]`` for a feature, ``reasons[1]`` for the label.  ``row`` and ``position`` stay."""
    from .engine import InvalidCellError
    is_label = e.position == len(fields)
    name = label if is_label else fields[e.position]
    return InvalidCellError(e.row, e.position, f"{call}: field {name!r} of the row with _id {ids[e.row]} {reasons[is_label]}")


class Features:
    """What :meth:`DeviceFrame.features` made: ``x[i]`` the feature matrix of shard i (one on a single GPU) as a
    zero-copy ``__cuda_array_interface__`` view of shape ``(n_i, len(fields))``, row-major, on ``devices[i]``
    (``torch.as_tensor(features.x[i], device=f"cuda:{features.devices[i]}")`` reads it in place); ``y[i]`` the label's
    vector of n_i values, or ``y`` None; ``row_ids`` the ``_id`` of every row, shards concatenated in order; ``fields``
    the column order.  Owns its tables and frees them in :meth:`release` (or with ``with``); keeps its frame alive."""

    def __init__(self, frame: DeviceFrame, parts, fields, label, dtype):
        import numpy as np
        self._frame, self._parts = frame, list(parts)
        self.fields, self.label, self.dtype = list(fields), label, dtype
        self.devices = [p.x.engine.device for p in self._parts]
        self.x = [p.matrix(keepalive=self) for p in self._parts]
        self.y = [p.vector(keepalive=self) for p in self._parts] if label is not None else None
        ids = np.asarray(frame.ids)
        self.row_ids = np.concatenate([ids[p.first:p.first + p.nkept] if p.kept is None else ids[p.rows]
                                       for p in self._parts]) if self._parts else np.zeros(0, np.int64)

    def release(self):
        parts, self._parts = self._parts, []
        for p in parts:
            p.free()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.release()


def device_frame(database, filename, engine, text: bool = False) -> DeviceFrame:
    """``Builder.__file_processor``'s frame (data rows, metadata columns dropped) handed over ON THE DEVICE: the
    numeric fields of the dataset as zero-copy views of the resident slabs (``builder_image/builder.py:172-194`` loads
    the same frame into Spark).  ``text``: the fields of the store that are text (:class:`~table_cache.Snapshot`'s rule;
    mixed fields stay out) join it as int32 dictionary codes made on the device from the resident text columns — the
    same columns ``/histograms`` counts, uploaded only when none is resident yet; the fields keep the store's order.
    Without ``text`` the frame holds the number fields alone — use :func:`file_processor` for the host form."""
    if getattr(database, "has_columns", lambda _f: False)(filename):
        names = [f for f in database.column_names(filename) if f not in METADATA_FIELDS]
        numeric = [f for f in names if getattr(database.column(filename, f), "kind", "") == "number"]
    else:
        names, rows = frame_fields(database, filename)
        numeric = [f for f in names if rows and columnar.numeric_column([d.get(f) for d in rows]) is not None]
    if not text:
        data = engine.resident.ensure(database, filename, numeric)
        return DeviceFrame(engine.resident, data, numeric)
    from .engine import text_dictionary
    from .table_cache import Snapshot
    snap = Snapshot(database, filename)
    words = [f for f in names if f not in numeric and snap.field(f).text is not None]
    data = engine.resident.ensure(database, filename, numeric, text=words, snapshot=snap)
    codes = {}
    try:
        for f in words:
            cells = data.texts[f]
            table = engine.table("i32", cells.n, 1)
            codes[f] = (table, None)             # freed below if its codes fail
            codes[f] = (table, text_dictionary(cells.arr, engine.text_codes(cells, table, 0)))
    except BaseException:
        for table, _dictionary in codes.values():
            table.free()
        engine.resident.release(data)
        raise
    return DeviceFrame(engine.resident, data, [f for f in names if f in numeric or f in codes], codes)


def _frame(fields, rows, packed, resident):
    import numpy as np
    import pyarrow as pa
    arrays, names = [], []
    for f in fields:
        if packed[f] is not None:
            col, valid, kind = packed[f]
            if resident is not None:
                col = resident.table.to_numpy(resident.column[f])            # the slab, back from HBM
            if kind == "int":
                arr = pa.array(np.where(valid, col, 0).astype(np.int64), mask=~valid)
            else:
                arr = pa.array(col, mask=~valid)
        else:
            arr = pa.array([None if d.get(f) is None else (d.get(f) if isinstance(d.get(f), str) else repr(d.get(f)))
                            for d in rows], type=pa.string())
        arrays.append(arr)
        names.append(f)
    return pa.table(arrays, names=names) if names else pa.table({})
