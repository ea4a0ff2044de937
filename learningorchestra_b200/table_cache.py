"""Datasets resident in HBM between requests.

In the reference every request re-reads the whole Mongo collection (Spark ``load`` in
``projection_image/projection.py:35-37``, one ``$group`` scan per field in
``histogram_image/histogram.py:31-36``).  Here the numeric columns of a dataset are packed once into a
columnar :class:`~learningorchestra_b200.engine.DeviceTable` and stay on the GPU: later histogram /
projection requests on the same dataset run on the resident slabs (``lo_project_cast_hist_dev``) with no
document scan and no host->device copy, which is the regime ``bench.py``'s ``value`` measures.

Text fields (every dataset arrives as text) are parsed on the device straight into their slabs with CPython's
``float()`` (``lo_parse_number_to_table``): a binned histogram or a ``castTo`` projection of a freshly uploaded CSV
needs no ``/fieldTypes`` job first, and the dataset is never modified.  The slab equals the one ``/fieldTypes
"number"`` would have led to, bit for bit.

Staleness: the in-process :class:`~learningorchestra_b200.utils.Database` bumps ``version(filename)`` on every
write to data rows; a cached table is used only while its version matches.  A ``Database`` without
``version`` (foreign object) is never cached.  Eviction: least recently used beyond ``max_bytes``.
"""
from __future__ import annotations

import threading
from collections import OrderedDict

import numpy as np

from . import columnar


class ResidentDataset:
    def __init__(self, version, ids, fields, kinds, nulls, table):
        self.version, self.ids, self.fields, self.kinds, self.nulls, self.table = version, ids, fields, kinds, nulls, table
        self.column = {f: i for i, f in enumerate(fields)}
        self.users = 0          # leases handed out and not yet released (guarded by ResidentTables._lock)
        self.retired = False    # dropped from the cache: freed when the last user releases it

    @property
    def nbytes(self) -> int:
        return self.table.pitch_bytes * self.table.ncols


def device_number_column(values: np.ndarray, valid: np.ndarray, is_int: np.ndarray):
    """(float64 slab, valid mask, "int" | "float") of a stored number column for the HBM-resident copy: nulls become NaN
    (the kernels skip them), a fully valid column is handed over as it is (no copy), and the int / float kind is read
    without materialising the valid subset.  Same result as ``np.where(valid, values, nan)`` / ``is_int[valid].all()``."""
    if valid.all():
        return values, valid, "int" if is_int.all() else "float"
    return np.where(valid, values, np.nan), valid, "int" if bool((is_int | ~valid).all()) else "float"


def _number_source(packed):
    return None if packed is None else ("number", packed)


def is_text_field(values) -> bool:
    """A document field the text route takes: at least one value, and every value that is not None a ``str``."""
    return any(v is not None for v in values) and all(v is None or type(v) is str for v in values)


def parse_text_column(engine, table, col: int, cells):
    """``float(cell)`` of every cell of a text field — an Arrow string array, or a list of ``str`` / None — parsed on
    the device straight into f64 column ``col`` of ``table`` (a ``DeviceTable`` or ``ShardedTable``): None and ``""``
    become NaN, every other cell the binary64 ``/fieldTypes "number"`` stores.  Returns (kind "int" | "float", null
    count).  The first bad cell in row order fails the call: ValueError with ``float()``'s message for text it rejects,
    RuntimeError for a cell over the parser's 1 MiB limit (there is no host fallback)."""
    chars, offsets, validity = columnar.text_buffers(columnar.number_text(cells))
    summary = engine.parse_number_into(table, col, chars, offsets, validity)
    bad = [r for r in (summary["first_invalid"], summary["first_unsupported"]) if r is not None]
    if bad:
        row = min(bad)
        cell = cells[row].as_py() if hasattr(cells, "to_pylist") else cells[row]
        if row == summary["first_unsupported"]:
            raise RuntimeError(f"cell of {len(cell)} characters exceeds the device parser's 1 MiB limit "
                               "and there is no CPU fallback")
        raise ValueError(f"could not convert string to float: {cell!r}")
    return ("int" if summary["integer"] else "float"), summary["nulls"]


class ResidentTables:
    def __init__(self, engine, max_bytes: int = 64 << 30):
        self.engine, self.max_bytes = engine, max_bytes
        self._entries: "OrderedDict[str, ResidentDataset]" = OrderedDict()
        self._lock = threading.RLock()
        self.hits = self.misses = 0

    def lease(self, database, filename: str, fields):
        """``with resident.lease(db, name, fields) as data:`` — the table cannot be freed (version bump, eviction,
        invalidate, another job's rebuild) while the block runs GPU work on it."""
        cache = self

        class _Lease:
            def __enter__(self_inner):
                self_inner.data = cache.ensure(database, filename, fields)
                return self_inner.data

            def __exit__(self_inner, *exc):
                cache.release(self_inner.data)
        return _Lease()

    def release(self, entry: ResidentDataset) -> None:
        with self._lock:
            entry.users -= 1
            if entry.retired and entry.users <= 0:
                entry.table.free()

    def _retire(self, entry: ResidentDataset) -> None:
        """Called with the lock held: free now if nobody uses the table, else when the last lease ends."""
        entry.retired = True
        if entry.users <= 0:
            entry.table.free()

    def ensure(self, database, filename: str, fields) -> ResidentDataset:
        """Resident table holding (at least) ``fields`` of ``filename``; built from the documents on a miss.
        A field may be numeric or text (a column-store text column, or document values that are all ``str`` / None):
        text is parsed on the device into its slab, the dataset itself stays text.  Raises ValueError if a requested
        field is neither, or names the first cell ``float()`` rejects; on any failure nothing is cached.  The returned
        entry is LEASED: pair every call with :meth:`release` (or use :meth:`lease`)."""
        version = database.version(filename) if hasattr(database, "version") else None
        with self._lock:
            entry = self._entries.get(filename)
            if entry is not None and version is not None and entry.version == version and all(f in entry.column for f in fields):
                self._entries.move_to_end(filename)
                self.hits += 1
                entry.users += 1
                return entry
            self.misses += 1
            keep = [f for f in (entry.fields if entry is not None and entry.version == version else []) if f not in fields]
            wanted = list(fields) + keep
            columnar_rows = getattr(database, "has_columns", lambda _f: False)(filename)
            if columnar_rows:            # rows already stored as columns (column_store): no document is touched
                row_ids = database.row_ids(filename)
                rows = row_ids
            else:
                rows = columnar.data_rows(database.find(filename, {}))
                rows.sort(key=lambda d: d["_id"])
                row_ids = np.array([d["_id"] for d in rows], dtype=np.int64)
            sources, names = [], []          # per resident column: ("number", packed) or ("text", cells)
            for f in wanted:
                if columnar_rows:
                    c = database.column(filename, f)
                    if c is not None and c.kind == "object":
                        src = _number_source(columnar.numeric_column(c.to_pylist()))
                    elif c is not None and c.kind == "number":
                        src = ("number", device_number_column(c.values, c.valid, c.is_int))
                    elif c is not None and c.kind == "text":
                        src = ("text", c.arr)
                    else:
                        src = None
                else:
                    values = [d.get(f) for d in rows]
                    src = _number_source(columnar.numeric_column(values))
                    if src is None and is_text_field(values):
                        src = ("text", values)
                if src is None:
                    if f in fields:
                        raise ValueError(f"field {f!r} is not numeric; run /fieldTypes first")
                    continue                 # a previously resident column that stopped being numeric: drop it
                names.append(f); sources.append(src)
            table = self.engine.table("f64", len(rows) if sources else 0, max(len(sources), 1))
            kinds, nulls = [], []
            try:
                for j, (how, src) in enumerate(sources):
                    if how == "number":
                        values, valid, kind = src
                        if len(rows):
                            table.upload(j, values)
                        kinds.append(kind); nulls.append(int(valid.size - np.count_nonzero(valid)))
                    else:
                        kind, n_null = parse_text_column(self.engine, table, j, src)
                        kinds.append(kind); nulls.append(n_null)
            except BaseException:
                table.free()                 # a bad cell: nothing of the partly built table stays, nothing is cached
                raise
            new = ResidentDataset(version, row_ids, names, kinds, nulls, table)
            new.users = 1
            if entry is not None:
                self._entries.pop(filename, None)
                self._retire(entry)
            if version is not None:
                self._entries[filename] = new
                self._entries.move_to_end(filename)
                self._evict()
            else:
                new.retired = True         # never cached (foreign Database without version()): freed on release
            return new

    def _evict(self):
        total = sum(e.nbytes for e in self._entries.values())
        while total > self.max_bytes and len(self._entries) > 1:
            _name, old = self._entries.popitem(last=False)
            total -= old.nbytes
            self._retire(old)

    def invalidate(self, filename: str) -> None:
        with self._lock:
            entry = self._entries.pop(filename, None)
            if entry is not None:
                self._retire(entry)

    def clear(self) -> None:
        with self._lock:
            for e in self._entries.values():
                self._retire(e)
            self._entries.clear()
