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

Text columns are kept as text too, next to the slabs in the same :class:`ResidentDataset`, for the ``$group`` of
``/histograms`` without ``bins`` (``Engine.text`` / ``lo_text_upload``): a column-store text column's Arrow buffers go
up as they are, a document-store text field's cells with None as null.  Such a column is never parsed, so a field of
words (``Sex``) is kept and counted like any other; the host keeps the Arrow array to read the group keys from, and the
entry records how many documents that are not data rows (the metadata document) lack the field — the ``null`` group.

Number fields are counted from their slabs (``Engine.value_counts_column``).  For each such field the entry records,
when it is built, whether the slab came from a number column of the store (a text field parsed for a binned request is
still counted as text), the documents that are not data rows lacking it, and how its keys are typed: a column store's
``integers_collapsed``, a document store's ``numeric_column`` kind.  A slab already resident for a binned or ``castTo``
request is counted as it is.  :class:`Snapshot` is the one reader of a dataset's fields, for this build and for
``Histogram``'s host route.

Staleness: the in-process :class:`~learningorchestra_b200.utils.Database` bumps ``version(filename)`` on every
write to data rows (a ``/fieldTypes`` job included); a cached entry is used only while its version matches, and the
next request rebuilds it.  A ``Database`` without ``version`` (foreign object) is never cached: its entry is freed when
the request's lease ends.  Eviction: least recently used beyond ``max_bytes``, slabs and text columns counted together.
"""
from __future__ import annotations

import threading
from collections import OrderedDict
from functools import cached_property
from typing import NamedTuple

import numpy as np

from . import columnar
from .column_store import large_text


class ResidentDataset:
    """One dataset's resident device objects.  An entry rebuilt at the same version shares the objects it does not
    change with its predecessor (each object counts the entries holding it, ``holders``) and a device object is freed
    with the last entry that holds it, so a lease on either entry keeps everything it reads alive."""

    def __init__(self, version, ids, fields, kinds, nulls, table, texts=None, absent=None, numbers=None, sources=None):
        self.version, self.ids, self.fields, self.kinds, self.nulls, self.table = version, ids, fields, kinds, nulls, table
        self.column = {f: i for i, f in enumerate(fields)}
        # text columns kept as text for $group: field -> DeviceText, or None for a field that was checked and is not a
        # text field (number, mixed, all null, or set on a document that is not a data row)
        self.texts = dict(texts or {})
        # number fields whose $group is counted from their slab: field -> whether a finite integral key is an int (the
        # host route's rule for that store), or None for a field that was checked and takes another route (text, even
        # when parsed into a slab for a binned request; mixed; set on a document that is not a data row)
        self.numbers = dict(numbers or {})
        self.absent = dict(absent or {})   # counted field -> documents that are not data rows and lack it (null group)
        # a column store's entry: ("slab" | "text", field) -> the store columns that object serves (the one it was made
        # from, and any that replaced it with the same values); None for a document store, whose entries serve one version
        self.sources = sources
        # objects handed over for store columns written after this entry was built: ("slab" | "text", field) ->
        # (column, object, kind, nulls) — a slab is a one-column table, kind and nulls as in ``kinds`` / ``nulls``
        self.adopted = {}
        self.users = 0          # leases handed out and not yet released (guarded by ResidentTables._lock)
        self.retired = False    # dropped from the cache: freed when the last user releases it
        for obj in self._objects():
            obj.holders = getattr(obj, "holders", 0) + 1

    def _objects(self):
        return [o for o in [self.table, *self.texts.values(), *(a[1] for a in self.adopted.values())] if o is not None]

    @property
    def nbytes(self) -> int:
        return sum(o.pitch_bytes * o.ncols if hasattr(o, "ncols") else o.nbytes for o in self._objects())

    def free(self) -> None:
        for obj in self._objects():
            obj.holders -= 1
            if obj.holders <= 0:
                obj.free()


def device_number_column(values: np.ndarray, valid: np.ndarray, is_int: np.ndarray):
    """(float64 slab, valid mask, "int" | "float") of a stored number column for the HBM-resident copy: nulls become NaN
    (the kernels skip them), a fully valid column is handed over as it is (no copy), and the int / float kind is read
    without materialising the valid subset.  Same result as ``np.where(valid, values, nan)`` / ``is_int[valid].all()``."""
    if valid.all():
        return values, valid, "int" if is_int.all() else "float"
    return np.where(valid, values, np.nan), valid, "int" if bool((is_int | ~valid).all()) else "float"


def is_text_field(values) -> bool:
    """A document field the text route takes: at least one value, and every value that is not None exactly a ``str``
    (no store holds a ``str`` subclass such as ``numpy.str_``; a field of them would count as mixed)."""
    return any(v is not None for v in values) and all(v is None or type(v) is str for v in values)


class _Field(NamedTuple):
    """What one field of a dataset is for the resident copy.  ``slab``: what its resident column is made from —
    ``("number", (values, valid, kind))`` to upload, ``("text", cells)`` to parse, or None (not numeric).  ``text``: the
    cells to keep as text for counting, or None.  ``as_int``: the key rule ``ResidentDataset.numbers`` records when its
    groups come from its slab, else None.  ``absent``: the documents that are not data rows and lack it."""
    slab: tuple | None
    text: object
    as_int: bool | None
    absent: int


class Values(NamedTuple):
    """A field as the host route counts it, ``data`` as the store has it: ``kind`` "number" (``numeric_column``'s values,
    valid mask and key kind), "text" (the cells, an Arrow array or a list), "mixed" (a list) or None (no value set).
    ``extra``: the Values of what documents that are not data rows set, or None.  ``nulls``: the null cells of ``data``
    and the documents that are not data rows and lack the field."""
    kind: str | None
    data: object
    extra: "Values | None"
    nulls: int


def classify(values) -> Values:
    """A list of document values by the document store's rule: text when every value that is not None is a ``str``,
    number when :func:`columnar.numeric_column` packs them, else mixed."""
    if is_text_field(values):
        return Values("text", values, None, sum(1 for v in values if v is None))
    packed = columnar.numeric_column(values)
    if packed is None:
        return Values("mixed", values, None, sum(1 for v in values if v is None))
    n = int(np.count_nonzero(packed[1]))
    return Values("number" if n else None, packed, None, len(values) - n)


class Snapshot:
    """The dataset as one request reads it: its version, the data rows (or the column store's handle), their ids and
    the documents that are not data rows.  The one place that says what kind a stored field is, for the resident build
    (:meth:`field`), for the host route (:meth:`values`) and for the cells a cast writes (:meth:`valid`).

    Only ``version`` is read up front, before any data, so an entry built from the snapshot is never newer than the
    version it records.  The rest is read on first use: a request the resident copy answers reads no document."""

    def __init__(self, database, filename: str):
        self.database, self.filename = database, filename
        self.version = database.version(filename) if hasattr(database, "version") else None
        self.columnar = getattr(database, "has_columns", lambda _f: False)(filename)
        self._fields, self._columns = {}, {}

    @cached_property
    def documents(self):
        return list(self.database.find(self.filename, {}))

    @cached_property
    def data(self):
        """A document store's data rows in the order the store holds them."""
        return columnar.data_rows(self.documents)

    @cached_property
    def rows(self):
        return sorted(self.data, key=lambda d: d["_id"])

    @cached_property
    def others(self):
        if self.columnar:        # rows stored as columns (column_store): no data row is materialised
            return self.database.other_documents(self.filename)
        return [d for d in self.documents if d.get("_id") == columnar.METADATA_DOCUMENT_ID]

    @cached_property
    def row_ids(self):
        if self.columnar:
            return self.database.row_ids(self.filename)
        return np.array([d["_id"] for d in self.rows], dtype=np.int64)

    def column(self, f):
        """A column store's column of ``f`` as this snapshot first read it (None when no data row has the field)."""
        if f not in self._columns:
            self._columns[f] = self.database.column(self.filename, f)
        return self._columns[f]

    def _absent(self, f) -> int:
        """The documents that are not data rows and lack ``f``: they count under ``null``."""
        return sum(1 for d in self.others if d.get(f) is None)

    def values(self, f) -> Values:
        """``f`` as the host route counts it: a document store's documents in store order, the other documents among
        them; a column store's column by its kind (an object column by :func:`classify`), with ``extra``."""
        if not self.columnar:
            return classify([d.get(f) for d in self.documents])
        c, n = self.column(f), len(self.row_ids)
        kind = c.kind if c is not None else None
        if kind == "number":
            key_kind = "int" if c.integers_collapsed else "float"
            v = Values("number", (c.values, c.valid, key_kind), None, n - int(np.count_nonzero(c.valid)))
        elif kind == "text":
            v = Values("text", c.arr, None, c.arr.null_count)
        else:
            v = classify(c.to_pylist()) if kind == "object" else Values(None, None, None, n)
        extra = [d[f] for d in self.others if d.get(f) is not None]
        return Values(v.kind if v.nulls < n else None, v.data, classify(extra) if extra else None,
                      v.nulls + self._absent(f))

    def field(self, f) -> _Field:
        """``f`` for the resident copy, from the data rows alone."""
        if f not in self._fields:
            slab = text = as_int = None
            if self.columnar:
                c = self.column(f)
                kind = c.kind if c is not None else None
                if kind == "number":
                    slab, as_int = ("number", device_number_column(c.values, c.valid, c.is_int)), c.integers_collapsed
                elif kind == "object":               # its groups are counted by the host route
                    v = classify(c.to_pylist())
                    slab = ("number", v.data) if v.kind not in ("text", "mixed") else None
                elif kind == "text":
                    slab, text = ("text", c.arr), c.arr
            else:
                v = classify([d.get(f) for d in self.rows])
                if v.kind == "text":
                    slab, text = ("text", v.data), v.data
                elif v.kind != "mixed":              # a number field, or one that no row sets
                    slab, as_int = ("number", v.data), v.data[2] == "int"
            absent = self._absent(f)
            if absent < len(self.others):
                text = as_int = None     # its groups are not the data rows' alone: the host route counts it
            self._fields[f] = _Field(slab, text, as_int, absent)
        return self._fields[f]

    def valid(self, f) -> np.ndarray:
        """One bool per data row, in :attr:`rows` order, of a field the resident copy holds: the cell holds a number
        after ``float()`` (not null, not ``""``).  A column store's number or text column is read as it is stored; the
        slab's copy of its values is never made here."""
        c = self.column(f) if self.columnar else None
        if c is not None and c.kind == "number":
            return c.valid
        if c is not None and c.kind == "text":
            return columnar.number_text_valid(c.arr)
        how, src = self.field(f).slab            # a document field or an object column: what the slab is made from
        return src[1] if how == "number" else columnar.number_text_valid(large_text(src))


class _Plan(NamedTuple):
    """What a miss builds: ``columns`` (field, slab) in table order, a slab as :class:`_Field` has it or ``("copy",
    (table, column, kind, nulls))`` for a resident slab copied device to device; or None when ``shared``'s table is used
    as it is.  ``uploads`` the text columns to make, field -> cells (None: recorded as not text); the rest as in
    ResidentDataset."""
    columns: list | None
    uploads: dict
    texts: dict
    numbers: dict
    absent: dict
    shared: "ResidentDataset | None" = None


def _carried(prev, snap: Snapshot):
    """What ``prev``, the cached entry of an older version, still holds for ``snap``: (texts field -> text column, slabs
    field -> (table, column, kind, nulls)).  A stored column is immutable (``set_column`` replaces the object), so an
    object made from store column ``c`` with row ids ``ids`` serves every later version whose snapshot still holds the
    same ``c`` and ``ids`` objects.  Nothing for a document store: its writes are per document and its fields may hold
    mixed cells, so its entries serve their own version only."""
    if prev is None or prev.sources is None or not snap.columnar or prev.ids is not snap.row_ids:
        return {}, {}

    def serves(role, f, made_from):
        return any(c is snap.column(f) for c in made_from.get((role, f), ()))

    texts = {f: t for f, t in prev.texts.items() if t is not None and serves("text", f, prev.sources)}
    slabs = {f: (prev.table, j, prev.kinds[j], prev.nulls[j]) for j, f in enumerate(prev.fields)
             if serves("slab", f, prev.sources)}
    for (role, f), (column, obj, kind, nulls) in prev.adopted.items():
        if column is snap.column(f):
            if role == "text":
                texts.setdefault(f, obj)
            else:
                slabs.setdefault(f, (obj, 0, kind, nulls))
    return texts, slabs


def _plan(base, prev, fields, text, numbers, snap: Snapshot) -> _Plan:
    """The entry a miss builds from ``snap``, given ``base``, the cached entry at the same version (or None): what
    ``base`` holds is shared, not built again — its text columns always, its table when no requested or counted number
    field is missing from it.  Without a base, ``prev`` (the stale entry, or None) gives what it still holds
    (:func:`_carried`): those text columns are taken as they are, those slabs copied device to device, or its whole
    table shared when it holds exactly the columns the entry needs.  Raises ValueError for the first requested field
    that is neither number nor text."""
    texts = dict(base.texts) if base else {}
    counted = dict(base.numbers) if base else {}
    absent = dict(base.absent) if base else {}
    kept_texts, kept_slabs = _carried(prev, snap) if base is None else ({}, {})
    resident = base.fields if base else list(kept_slabs)
    for f, t in kept_texts.items():
        if snap.field(f).text is not None:
            texts[f], absent[f] = t, snap.field(f).absent
    uploads = {}
    for f in dict.fromkeys(text):
        if f not in texts:
            uploads[f], absent[f] = snap.field(f).text, snap.field(f).absent
    grow = []                    # number fields to count that are not resident (every resident field is in counted)
    for f in dict.fromkeys(numbers):
        if f not in counted:
            counted[f], absent[f] = snap.field(f).as_int, snap.field(f).absent
            if counted[f] is not None and f not in resident:
                grow.append(f)
    if base and not grow and all(f in base.column for f in fields):
        return _Plan(None, uploads, texts, counted, absent, base)
    columns = []
    for f in [*fields, *(f for f in resident if f not in fields), *(f for f in grow if f not in fields)]:
        info = snap.field(f)
        counted[f] = info.as_int
        if info.as_int is not None:
            absent[f] = info.absent
        if info.slab is None:
            if f in fields:
                raise ValueError(f"field {f!r} is not numeric; run /fieldTypes first")
            continue                 # a previously resident column that stopped being numeric: drop it
        if info.slab[0] == "number":
            texts.setdefault(f, None)    # checked: not a text field, so a count request on it is a hit
        columns.append((f, ("copy", kept_slabs[f]) if f in kept_slabs else info.slab))
    if prev is not None and kept_slabs and [f for f, _ in columns] == prev.fields and \
            all(how == "copy" and src[:2] == (prev.table, j) for j, (_f, (how, src)) in enumerate(columns)):
        return _Plan(None, uploads, texts, counted, absent, prev)
    return _Plan(columns, uploads, texts, counted, absent)


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

    def lease(self, database, filename: str, fields, text=(), numbers=(), snapshot=None):
        """``with resident.lease(db, name, fields, text, numbers) as data:`` — the table and the text columns cannot be
        freed (version bump, eviction, invalidate, another job's rebuild) while the block runs GPU work on them."""
        cache = self

        class _Lease:
            def __enter__(self_inner):
                self_inner.data = cache.ensure(database, filename, fields, text, numbers, snapshot)
                return self_inner.data

            def __exit__(self_inner, *exc):
                cache.release(self_inner.data)
        return _Lease()

    def release(self, entry: ResidentDataset) -> None:
        with self._lock:
            entry.users -= 1
            if entry.retired and entry.users <= 0:
                entry.free()

    def _retire(self, entry: ResidentDataset) -> None:
        """Called with the lock held: free now if nobody uses the table, else when the last lease ends."""
        entry.retired = True
        if entry.users <= 0:
            entry.free()

    def ensure(self, database, filename: str, fields, text=(), numbers=(), snapshot=None) -> ResidentDataset:
        """Resident table holding (at least) ``fields`` of ``filename``; built from the documents on a miss.
        A field may be numeric or text (a column-store text column, or document values that are all ``str`` / None):
        text is parsed on the device into its slab, the dataset itself stays text.  Raises ValueError if a requested
        field is neither, or names the first cell ``float()`` rejects; on any failure nothing is cached.

        ``text``: fields to keep as text columns for counting (``entry.texts``), never parsed.  A field that is not a
        text field there is recorded as None and raises nothing: its caller takes another route.
        ``numbers``: fields to count from their slabs (``entry.numbers``): a number field of the store is made resident
        if it is not already (a slab of a binned or ``castTo`` request is used as it is); any other field is recorded
        as None and raises nothing.  The returned entry is LEASED: pair every call with :meth:`release` (or use
        :meth:`lease`).
        ``snapshot``: the caller's :class:`Snapshot` of ``filename``, so that what it reads besides the entry comes from
        the same read of the store; the entry is checked against, or built at, its version."""
        snap = snapshot if snapshot is not None else Snapshot(database, filename)
        version = snap.version
        with self._lock:
            entry = self._entries.get(filename)
            if entry is not None and version is not None and entry.version == version and \
                    all(f in entry.column for f in fields) and all(f in entry.texts for f in text) and \
                    all(f in entry.numbers for f in numbers):
                self._entries.move_to_end(filename)
                self.hits += 1
                entry.users += 1
                return entry
            self.misses += 1
            base = entry if entry is not None and entry.version == version else None
            new = self._build(version, snap, _plan(base, entry, fields, text, numbers, snap))
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

    def _build(self, version, snap: Snapshot, plan: _Plan) -> ResidentDataset:
        """The entry ``plan`` describes: its columns uploaded, parsed or copied in table order, then its text columns.  On
        any failure (a bad cell: the first in table order, so in request order) what this call made is freed and
        re-raised."""
        if plan.columns is None:
            table, names, kinds, nulls = plan.shared.table, plan.shared.fields, plan.shared.kinds, plan.shared.nulls
        else:
            names, kinds, nulls = [f for f, _slab in plan.columns], [], []
            table = self.engine.table("f64", len(snap.row_ids) if names else 0, max(len(names), 1))
        made = {}
        try:
            for j, (_f, (how, src)) in enumerate(plan.columns or ()):
                if how == "number":
                    values, valid, kind = src
                    if len(snap.row_ids):
                        table.upload(j, values)
                    kinds.append(kind); nulls.append(int(valid.size - np.count_nonzero(valid)))
                elif how == "copy":
                    from_table, from_col, kind, n_null = src
                    if len(snap.row_ids):
                        self.engine.copy_column(from_table, from_col, table, j)
                    kinds.append(kind); nulls.append(n_null)
                else:
                    kind, n_null = parse_text_column(self.engine, table, j, src)
                    kinds.append(kind); nulls.append(n_null)
            for f, cells in plan.uploads.items():
                made[f] = self.engine.text(cells) if cells is not None else None
        except BaseException:
            ResidentDataset(version, snap.row_ids, [], [], [], None if plan.columns is None else table, made).free()
            raise
        texts = {**plan.texts, **made}
        sources = None
        if snap.columnar:
            sources = {("slab", f): (snap.column(f),) for f in names}
            sources.update({("text", f): (snap.column(f),) for f, t in texts.items() if t is not None})
        return ResidentDataset(version, snap.row_ids, names, kinds, nulls, table, texts, plan.absent, plan.numbers,
                               sources)

    def adopt(self, filename: str, field: str, column, obj=None, slab=None, same_as=None) -> None:
        """Hand the cache the device result of a conversion that replaced column ``field`` of a column store by
        ``column``, so that the next miss takes it instead of building it from the host (:func:`_carried`).  ``obj``: a
        text column made from ``column``, or with ``slab`` = (kind, nulls) a one-column f64 table holding its values;
        None: the slab the cached entry made from column ``same_as`` (the one ``column`` replaced) holds them.  The cache owns ``obj`` from here on:
        it counts toward ``max_bytes`` and is freed with the entry it joins (invalidate, clear, eviction, the next
        version), or at once when there is no column-store entry to join."""
        with self._lock:
            entry = self._entries.get(filename)
            if entry is None or entry.sources is None:
                if obj is not None:
                    obj.free()
                return
            if obj is None:
                key = ("slab", field)
                if any(c is same_as for c in entry.sources.get(key, ())):
                    entry.sources[key] += (column,)
                return
            key = ("slab" if slab is not None else "text", field)
            obj.holders = getattr(obj, "holders", 0) + 1
            old = entry.adopted.pop(key, None)
            entry.adopted[key] = (column, obj, *(slab or (None, None)))
            if old is not None:
                old[1].holders -= 1
                if old[1].holders <= 0:
                    old[1].free()
            self._evict()

    def holding(self, database, filename: str, field: str, snapshot: "Snapshot") -> ResidentDataset | None:
        """The cached entry at ``snapshot``'s version when its table holds a slab of ``field``, LEASED (a hit: pair it
        with :meth:`release`); else None, and nothing is built."""
        with self._lock:
            entry = self._entries.get(filename)
            if entry is None or snapshot.version is None or entry.version != snapshot.version or field not in entry.column:
                return None
            self._entries.move_to_end(filename)
            self.hits += 1
            entry.users += 1
            return entry

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
