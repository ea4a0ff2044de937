"""``Projection`` — drop-in for ``projection_image/projection.py`` (same constructor, same ``create``).

Reference job (``projection.py:32-48``): Spark loads the input collection, drops ``_id == 0``, selects
``fields + ["_id"]``, appends the rows to the output collection, flips ``finished``.  Here the
``spark_session`` slot receives a :class:`~learningorchestra_b200.engine.Engine`.

* Plain request (reference schema): the select is pure data movement over documents and is done by the
  adapter — there is no arithmetic to put on a GPU, and the values must come back untouched (strings
  included).
* ``cast_to="float32"`` (this build's optional extension, REST key ``castTo``): the selected columns must
  be numeric or text (text is ``float(cell)`` parsed on the device; None / ``""`` stay None); they go through
  the fused sm_90a kernel (projection + fp64->fp32 RNE cast, and with
  ``bins`` a fixed-width histogram in the same pass) via ``lo_project_cast_hist_host``.
"""
from __future__ import annotations

from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import columnar
from .utils import Database, record_exception


class Projection:
    __FINISHED = "finished"
    __DOCUMENT_ID = "_id"
    __METADATA_FILE_ID = 0

    def __init__(self, metadata_creator, spark_session):
        self.__metadata_creator = metadata_creator
        self.__thread_pool = ThreadPoolExecutor()
        self.__engine = spark_session          # the slot the reference fills with a SparkSession
        self.last_job = None                   # Future of the submitted job (the reference drops it)

    def create(self, parent_filename: str, projection_filename: str, fields: list,
               database_url_input: str, database_url_output: str, cast_to: str | None = None,
               bins: int | None = None, value_range=None) -> None:
        self.__metadata_creator.create_file(projection_filename, parent_filename, fields)
        self.last_job = self.__thread_pool.submit(
            self.__execute_job, projection_filename, fields, database_url_input, database_url_output,
            cast_to, bins, value_range)

    def wait(self, timeout=None):
        if self.last_job is not None:
            self.last_job.result(timeout)

    def __execute_job(self, projection_filename, fields, database_url_input, database_url_output,
                      cast_to, bins, value_range) -> None:
        database = self.__metadata_creator.database_connector
        try:
            source = Database.collection_from_url(database_url_input)
            target = Database.collection_from_url(database_url_output)
            if getattr(database, "has_columns", lambda _f: False)(source):
                fields_with_id = self.__project_columns(database, source, target, list(fields), cast_to, bins, value_range)
                fields.append(self.__DOCUMENT_ID)        # projection.py:42 mutates the caller's list; kept
                del fields_with_id
                self.__metadata_creator.update_finished_flag(projection_filename, True)
                return
            rows = columnar.data_rows(database.find(source, {}))
            selected = list(fields)
            fields.append(self.__DOCUMENT_ID)       # projection.py:42 mutates the caller's list; kept
            ids = [d[self.__DOCUMENT_ID] for d in rows]
            if cast_to is None:
                out_docs = []
                for d in rows:
                    o = {f: d.get(f) for f in selected}
                    o[self.__DOCUMENT_ID] = d[self.__DOCUMENT_ID]
                    out_docs.append(o)
            elif cast_to == "float32":
                out_docs = self.__gpu_cast(database, target, rows, ids, selected, bins, value_range)
            else:
                raise ValueError(f"unknown cast_to {cast_to!r}")
            database.insert_many_in_file(target, out_docs)
            self.__metadata_creator.update_finished_flag(projection_filename, True)
        except BaseException as exc:                # reference: exception lost, finished stays False
            record_exception(database, projection_filename, exc)
            raise

    def __project_columns(self, database, source, target, selected, cast_to, bins, value_range):
        """``select(*fields, "_id")`` on a collection stored as columns (:mod:`column_store`): the output collection
        shares the selected column arrays (they are immutable) — no row is touched.  With ``cast_to="float32"`` the
        columns come from / go through the HBM-resident copy of the dataset and the fused kernel."""
        from .column_store import NumberColumn
        ids = database.row_ids(source)
        if cast_to is None:
            cols = {}
            for f in selected:
                c = database.column(source, f)
                cols[f] = c if c is not None else NumberColumn(np.full(ids.shape[0], np.nan), np.zeros(ids.shape[0], bool))
            database.create_table(target, ids, cols)
            return selected
        if cast_to != "float32":
            raise ValueError(f"unknown cast_to {cast_to!r}")
        if self.__engine is None:
            raise RuntimeError("cast_to needs an Engine in the spark_session slot (there is no CPU fallback)")
        with self.__engine.resident.lease(database, source, selected) as data:
            idx = [data.column[f] for f in selected]
            out = None
            try:
                if bins:
                    if value_range is None:
                        lo, hi = columnar.auto_range(*self.__engine.minmax_cast(data.table, idx), int(bins))
                    else:
                        lo = np.full(len(selected), value_range[0], np.float32)
                        hi = np.full(len(selected), value_range[1], np.float32)
                    out = self.__engine.table("f32", data.table.nrows, len(selected))
                    dev = self.__engine.project_cast_hist(data.table, idx, int(bins), lo, hi, out=out)
                    counts = dev.to_numpy()
                    dev.free()
                    database.update_one(target, {"histogram": {
                        f: {"bins": int(bins), "range": [float(lo[j]), float(hi[j])], "counts": [int(c) for c in counts[j]]}
                        for j, f in enumerate(selected)}}, {"_id": 0})
                else:
                    out = self.__engine.project_cast(data.table, idx)
                cols = {}
                for j, f in enumerate(selected):
                    src = database.column(source, f)
                    valid = columnar.number_text_valid(src.arr) if src.kind == "text" else src.valid
                    cols[f] = NumberColumn(np.where(valid, out.to_numpy(j).astype(np.float64), np.nan), valid)
            finally:
                if out is not None:
                    out.free()
        database.create_table(target, database.row_ids(source), cols)
        return selected

    def __gpu_cast(self, database, target, rows, ids, selected, bins, value_range):
        if self.__engine is None:
            raise RuntimeError("cast_to needs an Engine in the spark_session slot (there is no CPU fallback)")
        from .table_cache import is_text_field
        cols, masks = [], []
        for f in selected:
            values = [d.get(f) for d in rows]
            packed = columnar.numeric_column(values)
            if packed is None and is_text_field(values):
                packed = self.__parse_text(values)
            if packed is None:
                raise ValueError(f"field {f!r} is not numeric; run /fieldTypes first")
            cols.append(packed[0])
            masks.append(packed[1])
        n = len(rows)
        outs = [np.empty(n, dtype=np.float32) for _ in selected]
        counts = None
        if bins:
            if value_range is None:
                lo, hi = columnar.auto_range(*self.__engine.minmax_cast_host(cols), int(bins))
            else:
                lo = np.full(len(selected), value_range[0], np.float32)
                hi = np.full(len(selected), value_range[1], np.float32)
            counts, _ = self.__engine.project_cast_hist_host(cols, bins, lo, hi, out=outs)
            database.update_one(target, {"histogram": {
                f: {"bins": int(bins), "range": [float(lo[j]), float(hi[j])], "counts": [int(c) for c in counts[j]]}
                for j, f in enumerate(selected)}}, {"_id": 0})
        else:
            self.__engine.project_cast_hist_host(cols, None, out=outs)
        docs = []
        for i in range(n):
            o = {f: (float(outs[j][i]) if masks[j][i] else None) for j, f in enumerate(selected)}
            o[self.__DOCUMENT_ID] = ids[i]
            docs.append(o)
        return docs

    def __parse_text(self, values):
        """(float64 values, valid mask) of a text field: the cells parsed on the device by the same call the resident
        tables use (:func:`table_cache.parse_text_column`), then read back for the host pipeline."""
        from .table_cache import parse_text_column
        table = self.__engine.table("f64", len(values), 1)
        try:
            parse_text_column(self.__engine, table, 0, values)
            parsed = table.to_numpy(0)
        finally:
            table.free()
        return parsed, np.array([v is not None and v != "" for v in values], dtype=bool)
