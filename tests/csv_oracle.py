"""CPU oracle of the upload reader (test infrastructure): what the reference stores for a CSV body.

The reference reads ``POST /files`` with (``database_api_image/database.py:110-137``)::

    reader = csv.reader(codecs.iterdecode(response.iter_lines(), encoding="utf-8"), delimiter=",", quotechar='"')
    untreated_headers = next(reader)
    for row in reader: ...            # __treat_row: {headers[i]: row[i] for i in range(len(headers))}

:func:`csv_reference_rows` runs that same stdlib call on ``body.splitlines()``.  The rules it pins:

1. Lines.  A line ends at each run of ``\\r`` / ``\\n`` bytes, as ``bytes.splitlines()`` splits them, and
   ``iterdecode`` drops empty strings, so blank lines vanish — also inside a quoted field, after the last line and in
   ``\\r\\r``.  ``iter_lines`` yields the same lines: where a ``\\r\\n`` straddles one of its 512-byte chunks it
   yields one extra empty line, and that is dropped too.
2. Fields: CPython's ``_csv`` reader, default dialect (``strict=False``, no escapechar, no skipinitialspace).  A quote
   opens a field only at its start (``a"b`` stays ``a"b``, `` "x`` keeps its quote); ``""`` inside quotes is one quote;
   text after a closing quote is appended (``"ab"cd`` -> ``abcd``); a line break inside quotes is dropped and the record
   continues on the next line; an unterminated quote at EOF ends the record with what it has.  So every record ends
   at a line end or at EOF.
3. Field limit: 131 072 code points; the next one raises ``_csv.Error``.
4. UTF-8: strict, line by line (overlongs, surrogates, bytes >= 0xF5, truncated sequences raise UnicodeDecodeError at
   that line).  A BOM stays in the first header name (``\\W+`` removes it there).  A line that ends inside a multi-byte
   sequence is joined with the next line by the incremental decoder; that is not reproduced: such a body is
   reported as ``unsupported`` at the record of that line.
5. NUL: the reference image runs Python 3.7, whose ``_csv`` raises ``line contains NUL`` when it meets the character;
   3.11+ accept it.  Restated here: the line is handed to the reader only up to the NUL (so a field-limit error
   before it still wins), then the NUL is raised.  The default-dialect reader states, the field limit, and empty-line
   handling are otherwise the same in 3.7 and 3.12.
6. Rows.  Record 0 is the header and fixes ``ncols``; a data record with more fields keeps the first ``ncols``; one
   with fewer fails (IndexError in ``__treat_row``); an empty body fails (StopIteration from ``next(reader)``).
7. Failure.  Rules 3-6 end the same way: the data rows before the failing record are stored (``_id`` 1..k),
   ``finished`` stays False; a failing header stores nothing.
"""
from __future__ import annotations

import codecs
import csv

FIELD_LIMIT = 131072
KINDS = ("ok", "short_row", "field_limit", "bad_utf8", "nul", "unsupported", "empty")   # LO_CSV_* order


class _Stop(Exception):
    def __init__(self, kind):
        super().__init__(kind)
        self.kind = kind


def _lines(body: bytes, state: dict):
    """``codecs.iterdecode(body.splitlines(), "utf-8")`` with rules 4 and 5 made explicit."""
    for raw in body.splitlines():
        if not raw:
            continue
        dec = codecs.getincrementaldecoder("utf-8")()
        try:
            text = dec.decode(raw, False)
        except UnicodeDecodeError:
            raise _Stop("bad_utf8")
        if dec.getstate()[0]:
            raise _Stop("unsupported")
        k = text.find("\0")
        if k >= 0:
            state["nul"] = True
            yield text[:k]
            raise _Stop("nul")
        yield text


def csv_reference_rows(body: bytes):
    """(header, rows, failure): header = the header's cells (None when it fails), rows = the data rows stored (each cut
    to the header's width), failure = None or (kind, record index) with record 0 the header and kind in KINDS."""
    state = {"nul": False}
    reader = csv.reader(_lines(body, state), delimiter=",", quotechar='"')
    header, rows, index = None, [], 0
    try:
        for rec in reader:
            if state["nul"]:
                raise _Stop("nul")
            if index == 0:
                header = rec
            else:
                if len(rec) < len(header):
                    return header, rows, ("short_row", index)
                rows.append(rec[:len(header)])
            index += 1
    except _Stop as s:
        return (header if index else None), rows, (s.kind, index)
    except csv.Error as e:
        assert "field larger than field limit" in str(e), e
        return (header if index else None), rows, ("field_limit", index)
    if index == 0:
        return None, [], ("empty", 0)
    return header, rows, None
