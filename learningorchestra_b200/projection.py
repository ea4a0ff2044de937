"""``Projection`` — drop-in for ``projection_image/projection.py`` (same constructor, same ``create``).

Reference job (``projection.py:32-48``): Spark loads the input collection, drops ``_id == 0``, selects
``fields + ["_id"]``, appends the rows to the output collection, flips ``finished``.  Here the
``spark_session`` slot receives a :class:`~learningorchestra_b200.engine.Engine`.

* Plain request (reference schema): the select is pure data movement over documents and is done by the
  adapter — there is no arithmetic to put on a GPU, and the values must come back untouched (strings
  included).
* ``cast_to="float32"`` (this build's optional extension, REST key ``castTo``): the selected columns must
  be numeric or text (text is ``float(cell)`` parsed on the device; None / ``""`` stay None); on either store they are
  leased from the HBM-resident copy of the dataset (``table_cache``) and go through the fused sm_90a kernel
  (projection + fp64->fp32 RNE cast, and with ``bins`` a fixed-width histogram in the same pass).
"""
from __future__ import annotations

from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import columnar
from .column_store import NumberColumn
from .histogram import bins_result, binned
from .table_cache import Snapshot
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
            selected = list(fields)
            if getattr(database, "has_columns", lambda _f: False)(source):
                if cast_to is None:
                    self.__project_columns(database, source, target, selected)
                else:
                    self.__cast(database, source, target, selected, cast_to, bins, value_range)
                fields.append(self.__DOCUMENT_ID)        # projection.py:42 mutates the caller's list; kept
            elif cast_to is None:
                rows = columnar.data_rows(database.find(source, {}))
                fields.append(self.__DOCUMENT_ID)        # ... after the read, as the reference does
                out_docs = []
                for d in rows:
                    o = {f: d.get(f) for f in selected}
                    o[self.__DOCUMENT_ID] = d[self.__DOCUMENT_ID]
                    out_docs.append(o)
                database.insert_many_in_file(target, out_docs)
            else:
                fields.append(self.__DOCUMENT_ID)
                self.__cast(database, source, target, selected, cast_to, bins, value_range)
            self.__metadata_creator.update_finished_flag(projection_filename, True)
        except BaseException as exc:                # reference: exception lost, finished stays False
            record_exception(database, projection_filename, exc)
            raise

    def __project_columns(self, database, source, target, selected):
        """``select(*fields, "_id")`` on a collection stored as columns (:mod:`column_store`): the output collection
        shares the selected column arrays (they are immutable) — no row is touched."""
        ids = database.row_ids(source)
        cols = {}
        for f in selected:
            c = database.column(source, f)
            cols[f] = c if c is not None else NumberColumn(np.full(ids.shape[0], np.nan), np.zeros(ids.shape[0], bool))
        database.create_table(target, ids, cols)

    def __cast(self, database, source, target, selected, cast_to, bins, value_range):
        """``cast_to="float32"`` on either store: the selected columns come from / go through the HBM-resident copy of
        the dataset and the fused kernel, and one :class:`~table_cache.Snapshot` gives the slab, the row ids and which
        cells hold a number.  The histogram document is written first, then the rows: a column store's as columns, a
        document store's as documents in the order the store holds them."""
        if cast_to != "float32":
            raise ValueError(f"unknown cast_to {cast_to!r}")
        if self.__engine is None:
            raise RuntimeError("cast_to needs an Engine in the spark_session slot (there is no CPU fallback)")
        snap = Snapshot(database, source)
        with self.__engine.resident.lease(database, source, selected, snapshot=snap) as data:
            idx = [data.column[f] for f in selected]
            out = self.__engine.table("f32", data.table.nrows, len(selected)) if bins else None
            try:
                if bins:
                    lo, hi, counts = binned(self.__engine, data.table, idx, int(bins), value_range, out)
                    database.update_one(target, {"histogram": {f: bins_result(bins, lo[j], hi[j], counts[j])
                                                               for j, f in enumerate(selected)}}, {"_id": 0})
                else:
                    out = self.__engine.project_cast(data.table, idx)
                values = [out.to_numpy(j) for j in range(len(selected))]
            finally:
                if out is not None:
                    out.free()
        valid = [snap.valid(f) for f in selected]
        if snap.columnar:
            cols = {f: NumberColumn(np.where(ok, v.astype(np.float64), np.nan), ok)
                    for f, v, ok in zip(selected, values, valid)}
            database.create_table(target, snap.row_ids, cols)
            return
        # the slab is in _id order (Snapshot.rows): row k of the store's data rows is slab row at[k]
        ids = [d[self.__DOCUMENT_ID] for d in snap.data]
        at = np.empty(len(ids), np.int64)
        at[np.argsort(np.array(ids, np.int64), kind="stable")] = np.arange(len(ids))
        cells = []
        for v, ok in zip(values, valid):
            c = v[at].astype(object)             # Python floats
            c[~ok[at]] = None
            cells.append(c.tolist())
        keys = (*selected, self.__DOCUMENT_ID)
        database.insert_many_in_file(target, [dict(zip(keys, row)) for row in zip(*cells, ids)])
