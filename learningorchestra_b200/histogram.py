"""``Histogram`` — drop-in for ``histogram_image/histogram.py`` (same constructor and ``create_file``).

Reference job (``histogram.py:25-44``): per requested field one MongoDB pipeline
``[{"$group": {"_id": "$field", "count": {"$sum": 1}}}]`` over the WHOLE parent collection (metadata
document included: it has no such field, so it lands in — and inflates — the ``null`` group), one result
document ``{field: [{"_id": value, "count": n}, ...], "_id": k}`` per field, then ``finished: True``.

Here the counting runs on the GPU with no host dictionary:

* number fields (every value an int / float / None): GPU hash group-by on the binary64 keys
  (``lo_value_counts_f64_host``; -0.0 == 0.0, NaN == NaN as in MongoDB);
* text fields (every value a ``str`` / None): GPU hash group-by on the cells' bytes (``lo_value_counts_str_host``);
* mixed-type fields: the same byte-wise group-by over a tagged encoding under which two cells are equal exactly
  when MongoDB groups them (:func:`columnar.tagged_cell`: 1 == 1.0, ``True`` != 1, ``"1"`` != 1).

``None`` / missing values (the metadata document among them) are counted while packing.  With ``bins`` (optional
extension, REST keys ``bins`` / ``range``) the fields must be numeric and get the fixed-width B-semantics histogram
of SURVEY.md §8c from the fused kernel, run on the HBM-resident copy of the dataset (``table_cache``).
The dictionary-code kernels (``hist_u8_cols_host`` / ``value_counts_u32_host``) remain available on the engine for
columns that arrive already encoded (e.g. the uint8 tables of config M).
"""
from __future__ import annotations

import math
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import columnar
from .utils import record_exception


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
            if bins:
                results = self.__binned(parent_filename, fields, int(bins), value_range)
            elif getattr(self.database_connector, "has_columns", lambda _f: False)(parent_filename):
                results = self.__value_counts_columnar(parent_filename, fields)
            else:
                # unfiltered, like $group; materialised once (a pymongo Cursor can be walked only once)
                documents = list(self.database_connector.find(parent_filename, {}))
                results = self.__value_counts(documents, fields)
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
    def __value_counts(self, documents, fields):
        results = {}
        for f in fields:
            values = [d.get(f) for d in documents]
            present = [i for i, v in enumerate(values) if v is not None]
            packed = columnar.numeric_column(values) if documents else None
            if not present:
                groups = []
            elif packed is not None:                                     # number field: group-by on binary64 keys
                col, valid, kind = packed
                keys, counts = self.engine.value_counts_f64_host(col[valid])
                groups = [{"_id": (int(k) if kind == "int" else float(k)), "count": int(c)} for k, c in zip(keys, counts)]
            else:                                                        # text or mixed: group-by on the cells' bytes
                if all(isinstance(values[i], str) for i in present):
                    cells = [values[i] for i in present]
                else:
                    cells = [columnar.tagged_cell(values[i]) for i in present]
                rep, counts = self.engine.value_counts_str_host(cells)
                groups = [{"_id": values[present[int(r)]], "count": int(c)} for r, c in zip(rep, counts)]
            if len(present) != len(values):                              # None / missing (metadata document included)
                groups.append({"_id": None, "count": len(values) - len(present)})
            results[f] = groups
        return results

    def __value_counts_columnar(self, parent_filename, fields):
        """The same ``$group`` on a collection whose rows are stored as columns (:mod:`column_store`): a text field's
        Arrow buffers (chars + offsets) go to the byte-wise GPU group-by untouched, a number field's float64 array to
        the binary64 group-by — no document is materialised.  Documents that are not data rows (the metadata document)
        have none of the fields and count under ``null``, as in the reference."""
        db = self.database_connector
        others = db.other_documents(parent_filename)
        nrows = db.nrows(parent_filename)
        results = {}
        for f in fields:
            col = db.column(parent_filename, f)
            none_count = sum(1 for d in others if d.get(f) is None)
            extra = [d[f] for d in others if d.get(f) is not None]
            if col is None:
                groups, none_count = [], none_count + nrows
            elif col.kind == "number":
                keys, counts = self.engine.value_counts_f64_host(col.values[col.valid]) if col.valid.any() else ([], [])
                as_int = col.integers_collapsed
                groups = [{"_id": (int(k) if as_int and math.isfinite(k) and float(k).is_integer() else float(k)), "count": int(c)}
                          for k, c in zip(keys, counts)]
                none_count += int((~col.valid).sum())
            elif col.kind == "text":
                arr = col.arr.drop_null() if col.arr.null_count else col.arr
                none_count += col.arr.null_count
                from .column_store import TextColumn
                chars, offsets, _ = TextColumn(arr).packed()
                rep, counts = self.engine.value_counts_str_packed(chars, offsets)
                keys = arr.take(__import__("pyarrow").array(rep, type=__import__("pyarrow").int64())).to_pylist() if len(rep) else []
                groups = [{"_id": k, "count": int(c)} for k, c in zip(keys, counts)]
            else:                                    # mixed-type column: the document path's tagged byte-wise group-by
                sub = self.__value_counts([{f: v} for v in col.to_pylist()], [f])[f]
                none_count += sum(g["count"] for g in sub if g["_id"] is None)
                groups = [g for g in sub if g["_id"] is not None]
            if extra:                                # (result documents with the field: not produced by this stack)
                merged = self.__value_counts([{f: v} for v in extra], [f])[f]
                index = {columnar.group_key(g["_id"]): g for g in groups}
                for g in merged:
                    hit = index.get(columnar.group_key(g["_id"]))
                    if hit:
                        hit["count"] += g["count"]
                    else:
                        groups.append(g)
            if none_count:
                groups.append({"_id": None, "count": none_count})
            results[f] = groups
        return results

    # ---- B-semantics: fixed-width bins of the fp32-cast value -----------------------------------------
    def __binned(self, parent_filename, fields, bins, value_range):
        """Columns come from the GPU-resident copy of the dataset (built from the documents on first use,
        reused until the collection is written to): no document scan, no H2D on a repeat request."""
        with self.engine.resident.lease(self.database_connector, parent_filename, fields) as data:
            cols = [data.column[f] for f in fields]            # nulls are NaN in the slabs: skipped by the kernel
            if value_range is None:
                lo, hi = columnar.auto_range(*self.engine.minmax_cast(data.table, cols), bins)   # constant / empty columns included
            else:
                lo = np.full(len(fields), value_range[0], np.float32)
                hi = np.full(len(fields), value_range[1], np.float32)
            dev_counts = self.engine.project_cast_hist(data.table, cols, bins, lo, hi)
            counts = dev_counts.to_numpy()
            dev_counts.free()
        return {f: {"bins": bins, "range": [float(lo[j]), float(hi[j])], "counts": [int(c) for c in counts[j]]}
                for j, f in enumerate(fields)}
