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
