"""``Histogram`` — drop-in for ``histogram_image/histogram.py`` (same constructor and ``create_file``).

Reference job (``histogram.py:25-44``): per requested field one MongoDB pipeline
``[{"$group": {"_id": "$field", "count": {"$sum": 1}}}]`` over the WHOLE parent collection (metadata
document included: it has no such field, so it lands in — and inflates — the ``null`` group), one result
document ``{field: [{"_id": value, "count": n}, ...], "_id": k}`` per field, then ``finished: True``.

Here the counting runs on the GPU with no host dictionary:

* number fields (every value an int / float / None): GPU hash group-by on the binary64 keys (-0.0 == 0.0, NaN == NaN
  as in MongoDB) over the field's slab kept resident in HBM (``table_cache``, ``lo_value_counts_f64_table``; a slab
  already made resident by a binned or ``castTo`` request is counted as it is), leased with the text columns.  Nulls
  are NaN in the slab: the NaN key's count less the null rows is the group of real NaNs, and the ``null`` group is the
  null rows plus the documents that are not data rows.  Keys are typed by the store's rule, which ``table_cache``
  applies.  A rank group's process holds only its own rows, and a field set on a document that is not a data row is
  not in the slab: both take the host route;
* text fields (every value a ``str`` / None — every field of a fresh ``POST /files`` upload): GPU hash group-by on the
  cells' bytes over the field's text column kept resident in HBM (``table_cache``, ``lo_value_counts_text``), leased
  for the request.  The first request uploads the column; later ones copy no cell to the device and read no document.
  Group keys are read from the host's Arrow array at the representative rows; the ``null`` group is the column's null
  cells plus the documents that are not data rows (the metadata document);
* mixed-type fields: the byte-wise group-by over a tagged encoding under which two cells are equal exactly
  when MongoDB groups them (:func:`columnar.tagged_cell`: 1 == 1.0, ``True`` != 1, ``"1"`` != 1).

What HBM does not count takes the one host route, on either store: one :class:`~table_cache.Snapshot` reads the
dataset and says what each field is (``Snapshot.values``), and its values are packed per request — a number field's
valid values to ``lo_value_counts_f64_host``, a text field's non-null cells or a mixed field's tagged cells to
``lo_value_counts_str_host``.  ``None`` / missing values are counted by the reader.  With ``bins`` (optional
extension, REST keys ``bins`` / ``range``) the fields must be numeric or text (text is parsed with ``float()`` on the
device into the resident slab; the dataset stays text) and get the fixed-width B-semantics histogram of SURVEY.md §8c
from the fused kernel, run on the HBM-resident copy of the dataset (``table_cache``).
The dictionary-code kernels (``hist_u8_cols_host`` / ``value_counts_u32_host``) remain available on the engine for
columns that arrive already encoded (e.g. the uint8 tables of config M).
"""
from __future__ import annotations

import math
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import columnar
from .column_store import TextColumn, large_text
from .table_cache import Snapshot
from .utils import record_exception


def text_groups(arr, rep, counts, none_count):
    """Result groups of a text field counted on the device: the key of each group is the cell at its representative row
    of ``arr`` (the array that was counted, nulls included or not), then the ``null`` group of ``none_count`` null /
    missing cells when there are any."""
    import pyarrow as pa
    keys = arr.take(pa.array(np.asarray(rep, dtype=np.int64))).to_pylist() if len(rep) else []
    groups = [{"_id": k, "count": int(c)} for k, c in zip(keys, counts)]
    if none_count:
        groups.append({"_id": None, "count": int(none_count)})
    return groups


def number_groups(keys, counts, as_int, nulls, absent):
    """Result groups of a number field counted on the device.  Counted from its slab, where a null row is NaN: the NaN
    key's count less the ``nulls`` null rows is the group of real NaNs (emitted when there are any), and the ``null``
    group is those null rows plus the ``absent`` documents that are not data rows and lack the field.  The host route
    counts only the values that are not null and passes 0 for both.  ``as_int``: a finite integral key is an ``int``
    (the store's rule, which :class:`~table_cache.Snapshot` applies)."""
    groups = []
    for k, c in zip(np.asarray(keys, np.float64).tolist(), np.asarray(counts, np.uint64).tolist()):
        if math.isnan(k):
            c -= nulls
            if c <= 0:
                continue
        elif as_int and math.isfinite(k) and k.is_integer():
            k = int(k)
        groups.append({"_id": k, "count": int(c)})
    if nulls + absent:
        groups.append({"_id": None, "count": int(nulls + absent)})
    return groups


def binned(engine, table, cols, bins, value_range, out=None):
    """The fixed-width histogram of columns ``cols`` of a leased resident ``table``: (lo, hi, counts [k, bins]).  The
    range is ``value_range`` or, without one, the device min / max pre-pass's (constant and empty columns included);
    nulls are NaN in the slabs and skipped.  ``out``: an f32 table the fused kernel also writes the cast columns to."""
    if value_range is None:
        lo, hi = columnar.auto_range(*engine.minmax_cast(table, cols), bins)
    else:
        lo = np.full(len(cols), value_range[0], np.float32)
        hi = np.full(len(cols), value_range[1], np.float32)
    dev = engine.project_cast_hist(table, cols, bins, lo, hi, out=out)
    counts = dev.to_numpy()
    dev.free()
    return lo, hi, counts


def bins_result(bins, lo, hi, counts):
    """The result of one field's fixed-width histogram."""
    return {"bins": int(bins), "range": [float(lo), float(hi)], "counts": [int(c) for c in counts]}


class Histogram:
    METADATA_DOCUMENT_ID = 0
    DOCUMENT_ID_NAME = "_id"

    def __init__(self, database_connector, metadata_handler, engine=None):
        self.database_connector = database_connector
        self.metadata_handler = metadata_handler
        self.thread_pool = ThreadPoolExecutor()
        self.engine = engine
        self.last_job = None

    def create_file(self, parent_filename, histogram_filename, fields, bins=None, value_range=None):
        self.metadata_handler.create_file(parent_filename, histogram_filename, fields)
        self.last_job = self.thread_pool.submit(self.file_processing, parent_filename, histogram_filename, fields,
                                                bins, value_range)

    def wait(self, timeout=None):
        if self.last_job is not None:
            self.last_job.result(timeout)

    def file_processing(self, parent_filename, histogram_filename, fields, bins=None, value_range=None):
        try:
            if self.engine is None:
                raise RuntimeError("Histogram needs an Engine: the counting has no CPU fallback")
            snap = Snapshot(self.database_connector, parent_filename)     # one read of the dataset for every route
            if bins:
                results = self.__binned(snap, fields, int(bins), value_range)
            else:
                results = self.__value_counts_resident(snap, fields)
                rest = [f for f in fields if f not in results]
                if rest:
                    results.update(self.__value_counts_host(snap, rest))
            document_id = 1
            for field in fields:
                self.database_connector.insert_one_in_file(
                    histogram_filename, {field: results[field], self.DOCUMENT_ID_NAME: document_id})
                document_id += 1
            self.metadata_handler.update_finish_flag(histogram_filename, True)
        except BaseException as exc:
            record_exception(self.database_connector, histogram_filename, exc)
            raise

    # ---- R-semantics: exact value counts -------------------------------------------------------------
    def __value_counts_resident(self, snap, fields):
        """``$group`` of the fields that are text or number in the store, from their columns resident in HBM
        (``table_cache``), under one lease: the values cross PCIe when the column is first made resident, not on every
        request.  Returns the groups of those fields only; the others (mixed-type, set on a document that is not a data
        row) are left to the host route (``__value_counts_host``), and so is every number field of a rank group, whose
        process holds only its own rows."""
        resident = getattr(self.engine, "resident", None)
        if resident is None:
            return {}
        text = fields if getattr(self.engine, "value_counts_text", None) is not None else ()
        all_rows = getattr(self.engine, "world", 1) == getattr(self.engine, "nlocal", 1)
        numbers = fields if all_rows and getattr(self.engine, "value_counts_column", None) is not None else ()
        if not text and not numbers:
            return {}
        results = {}
        with resident.lease(self.database_connector, snap.filename, (), text=text, numbers=numbers,
                            snapshot=snap) as data:
            for f in fields:
                if f in results:
                    continue
                txt, as_int = data.texts.get(f), data.numbers.get(f)
                if txt is not None:
                    rep, counts = self.engine.value_counts_text(txt)
                    results[f] = text_groups(txt.arr, rep, counts, txt.nulls + data.absent[f])
                elif as_int is not None and f in data.column:
                    j = data.column[f]
                    keys, counts = self.engine.value_counts_column(data.table, j)
                    results[f] = number_groups(keys, counts, as_int, data.nulls[j], data.absent[f])
        return results

    def __value_counts_host(self, snap, fields):
        """The same ``$group`` read from the request's :class:`~table_cache.Snapshot`, packed per request.  What documents
        that are not data rows set is counted the same way and merged by :func:`columnar.group_key`; the ``null`` group
        is last."""
        results = {}
        for f in fields:
            values, groups = snap.values(f), {}
            for g in self.__groups(values) + (self.__groups(values.extra) if values.extra else []):
                hit = groups.setdefault(columnar.group_key(g["_id"]), g)
                if hit is not g:
                    hit["count"] += g["count"]
            results[f] = list(groups.values()) + ([{"_id": None, "count": values.nulls}] if values.nulls else [])
        return results

    def __groups(self, values):
        """The groups of the values of a :class:`~table_cache.Values` that are not null."""
        if values.kind == "number":
            col, valid, kind = values.data
            return number_groups(*self.engine.value_counts_f64_host(col[valid]), kind == "int", 0, 0)
        if values.kind == "text":
            arr = large_text(values.data)
            arr = arr.drop_null() if arr.null_count else arr
            chars, offsets, _ = TextColumn(arr).packed()
            return text_groups(arr, *self.engine.value_counts_str_packed(chars, offsets), 0)
        if values.kind == "mixed":
            present = [v for v in values.data if v is not None]
            rep, counts = self.engine.value_counts_str_host([columnar.tagged_cell(v) for v in present])
            return [{"_id": present[int(r)], "count": int(c)} for r, c in zip(rep, counts)]
        return []

    # ---- B-semantics: fixed-width bins of the fp32-cast value -----------------------------------------
    def __binned(self, snap, fields, bins, value_range):
        """Columns come from the GPU-resident copy of the dataset (built from the documents on first use,
        reused until the collection is written to): no document scan, no H2D on a repeat request."""
        with self.engine.resident.lease(self.database_connector, snap.filename, fields, snapshot=snap) as data:
            lo, hi, counts = binned(self.engine, data.table, [data.column[f] for f in fields], bins, value_range)
        return {f: bins_result(bins, lo[j], hi[j], counts[j]) for j, f in enumerate(fields)}
