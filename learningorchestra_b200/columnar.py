"""Documents <-> columns: the adapter either side of the GPU path.

The reference's table is one Mongo document per row (``database_api_image/database.py:124-137``);
the kernels want one contiguous slab per column.  This module does only that reshaping (plus the
dictionary encoding that turns arbitrary keys into dense codes) — never the arithmetic.
"""
from __future__ import annotations

import math

import numpy as np

METADATA_DOCUMENT_ID = 0
_EXACT_INT = 2 ** 53


def data_rows(documents):
    """``dataframe.filter(dataframe["_id"] != 0)`` (``projection.py:38-40``)."""
    return [d for d in documents if d.get("_id") != METADATA_DOCUMENT_ID]


def numeric_column(values):
    """(float64 array with NaN at nulls, valid mask, kind) or None if the column is not numeric.
    kind "int": every non-null value is an int that float64 holds exactly; "float": ints and floats mixed
    (what the Mongo-Spark connector's schema inference widens to double).

    Large columns are classified and packed by Arrow's C++ type inference; anything it does not take
    (mixed bool / int, huge ints, exotic objects) falls through to the per-value loop, which is the definition."""
    if len(values) >= 64:
        fast = _numeric_column_arrow(values)
        if fast is not NotImplemented:
            return fast
    return _numeric_column_loop(values)


def _numeric_column_arrow(values):
    try:
        import pyarrow as pa
        import pyarrow.compute as pc
        arr = pa.array(values)
    except Exception:                          # ArrowInvalid / ArrowTypeError / OverflowError: let the loop decide
        return NotImplemented
    t, n = arr.type, len(arr)
    if pa.types.is_null(t):
        return np.full(n, math.nan), np.zeros(n, dtype=bool), "int"
    if pa.types.is_integer(t):
        mm = pc.min_max(arr)
        lo, hi = mm["min"].as_py(), mm["max"].as_py()
        if lo is not None and (abs(lo) > _EXACT_INT or abs(hi) > _EXACT_INT):
            return None
        kind = "int"
    elif pa.types.is_floating(t):
        kind = "float"
    else:
        return None if (pa.types.is_string(t) or pa.types.is_boolean(t) or pa.types.is_large_string(t)) else NotImplemented
    valid = ~np.asarray(arr.is_null().to_numpy(zero_copy_only=False), dtype=bool)
    out = np.asarray(pc.cast(arr, pa.float64()).fill_null(math.nan).to_numpy(zero_copy_only=False), dtype=np.float64)
    return np.ascontiguousarray(out), valid, kind


def _numeric_column_loop(values):
    n = len(values)
    out = np.empty(n, dtype=np.float64)
    valid = np.ones(n, dtype=bool)
    all_int = True
    for i, v in enumerate(values):
        if v is None:
            out[i] = math.nan
            valid[i] = False
        elif isinstance(v, bool):
            return None
        elif isinstance(v, int):
            if abs(v) > _EXACT_INT:
                return None
            out[i] = float(v)
        elif isinstance(v, float):
            all_int = False
            out[i] = v
        else:
            return None
    return out, valid, ("int" if all_int else "float")


def _bin_width_f32(lo, hi, nbins: int):
    """(hi - lo) / nbins in fp32 round-to-nearest, as the histogram kernels compute it."""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.float32(np.float32(np.float32(hi) - np.float32(lo)) / np.float32(nbins))


def _f32_key(x) -> int:
    """An integer that orders fp32 values as numbers do (-0.0 and +0.0 share 0)."""
    b = int(np.float32(x).view(np.uint32))
    return b if b < 0x80000000 else -(b & 0x7FFFFFFF)


def _f32_of_key(k: int):
    return np.uint32(k if k >= 0 else 0x80000000 | -k).view(np.float32)


def auto_range(mins, maxs, nfinite, nbins: int):
    """[lo, hi] per column for a ``nbins``-bin request without ``range``, from the device's min / max / finite-count
    pre-pass.  Degenerate cases get a usable range instead of failing the job:

    * no finite value: [0, 1], as numpy.histogram does for empty input;
    * constant column v: [v - 0.5, v + 0.5] in fp32, numpy's rule.  Where 0.5 is below half an ulp (|v| >= 2^24) an edge
      moves to the neighbouring fp32 value instead.  Where that neighbour overflows (v = +-FLT_MAX) the edge stays at v
      and the other edge is the inward neighbour: the closed last (first) bin still holds v;
    * (hi - lo) / nbins rounds to 0 in fp32 (min and max a few subnormals apart): hi rises to the smallest fp32 value for
      which the width is positive.  The bins are about one subnormal ulp wide and max stays inside the range.

    Where hi - lo overflows fp32 (e.g. min -3e38, max 3e38) no finite fp32 range has that width; [min, max] is returned
    unchanged and the histogram call rejects it."""
    nbins = int(nbins)
    lo = np.array(mins, dtype=np.float32)
    hi = np.array(maxs, dtype=np.float32)
    inf = np.float32(np.inf)
    for j in range(lo.shape[0]):
        if int(nfinite[j]) == 0:
            lo[j], hi[j] = 0.0, 1.0
            continue
        if lo[j] == hi[j]:
            v = lo[j]
            a, b = np.float32(v - np.float32(0.5)), np.float32(v + np.float32(0.5))
            with np.errstate(over="ignore"):
                a = a if a != v else np.nextafter(v, -inf, dtype=np.float32)
                b = b if b != v else np.nextafter(v, inf, dtype=np.float32)
            if np.isinf(b):
                b = v
            if np.isinf(a):
                a = v
            lo[j], hi[j] = a, b
        if _bin_width_f32(lo[j], hi[j], nbins) == 0:
            # start above the answer (a width of one whole subnormal ulp per bin), then bisect on the ordered fp32 values
            good = np.float32(float(lo[j]) + nbins * 2.0 ** -149)
            while _bin_width_f32(lo[j], good, nbins) == 0:
                good = np.nextafter(good, inf, dtype=np.float32)
            bad_k, good_k = _f32_key(hi[j]), _f32_key(good)
            while good_k - bad_k > 1:
                mid = (good_k + bad_k) // 2
                if _bin_width_f32(lo[j], _f32_of_key(mid), nbins) > 0:
                    good_k = mid
                else:
                    bad_k = mid
            hi[j] = _f32_of_key(good_k)
    return lo, hi


def group_key(value):
    """Canonical key under MongoDB ``$group`` equality: numbers by value across int / float (1 == 1.0,
    -0.0 == 0.0), NaN with NaN, null and missing together, booleans apart from numbers, strings bytewise."""
    if value is None:
        return ("null",)
    if isinstance(value, bool):
        return ("bool", value)
    if isinstance(value, (int, float)):
        if isinstance(value, float):
            if math.isnan(value):
                return ("num", "nan")
            if math.isinf(value):
                return ("num", "inf" if value > 0 else "-inf")
            if value.is_integer():
                return ("num", int(value))
        return ("num", value)
    if isinstance(value, str):
        return ("str", value)
    return ("other", repr(value))


def ascii_number_text(cell: str) -> str:
    """What CPython's ``float(str)`` parses: ``_PyUnicode_TransformDecimalAndSpaceToASCII`` maps every non-ASCII
    character — Unicode whitespace to ``' '``, Unicode decimal digits (``"１２"``, ``"٣.٥"``) to ASCII digits,
    anything else makes the text invalid (``'?'``) — and leaves ASCII characters alone
    (``data_type_handler_image/data_type_update.py:40`` relies on it).  Code-point property lookups, not arithmetic:
    done here while the column is packed; the parse itself runs on the GPU."""
    if cell.isascii():
        return cell
    import unicodedata
    out = []
    for ch in cell:
        if ord(ch) < 128:
            out.append(ch)
        elif ch.isspace():
            out.append(" ")
        else:
            d = unicodedata.decimal(ch, None)
            if d is None:
                out.append("?")
                break
            out.append(chr(48 + d))
    return "".join(out)


def number_text(cells):
    """The text the number parser reads: an Arrow ``large_string`` array of ``cells`` (an Arrow string array, or a list
    of ``str`` / None) in which every cell with a non-ASCII character is :func:`ascii_number_text` of it (rare; found
    with one vectorised Arrow pass); nulls stay null.  An Arrow array that is all ASCII comes back as it is, same
    buffers.  Both ``/fieldTypes "number"`` and the text route of binned / cast requests use this one rule."""
    import pyarrow as pa
    import pyarrow.compute as pc
    from .column_store import large_text
    arr = large_text(cells)
    bad = pc.invert(pc.string_is_ascii(arr)).fill_null(False)
    if not pc.any(bad).as_py():
        return arr
    values = arr.to_pylist()
    for i in np.flatnonzero(np.asarray(bad.to_numpy(zero_copy_only=False), dtype=bool)):
        values[i] = ascii_number_text(values[i])
    return pa.array(values, type=pa.large_string())


def text_buffers(arr):
    """(chars uint8, offsets int64[n+1], validity) of an Arrow ``large_string`` array: views of its buffers, no copy.
    The offsets are the array's own (offsets[0] != 0 for a slice; cell i is chars[offsets[i]:offsets[i + 1]]);
    validity is None without nulls, else ``(bitmap uint8, bit_offset)`` — Arrow's validity bitmap and the first cell's
    bit in it."""
    n = len(arr)
    bufs = arr.buffers()
    offsets = np.frombuffer(bufs[1], dtype=np.int64, count=n + 1 + arr.offset)[arr.offset:] if n else np.zeros(1, np.int64)
    chars = np.frombuffer(bufs[2], dtype=np.uint8) if bufs[2] is not None and bufs[2].size else np.zeros(1, dtype=np.uint8)
    validity = (np.frombuffer(bufs[0], dtype=np.uint8), arr.offset) if arr.null_count and bufs[0] is not None else None
    return chars, offsets, validity


def zero_based(chars, offsets):
    """(chars, offsets) of :func:`text_buffers` with offsets[0] == 0, the layout ``lo_value_counts_str_host`` takes:
    chars from the first cell's first byte on (a view) and the offsets less offsets[0] (a copy, for a slice only)."""
    first = int(offsets[0])
    return (chars, offsets) if first == 0 else (chars[first:], offsets - first)


def number_text_valid(arr) -> np.ndarray:
    """bool per cell of an Arrow text array: the cell holds a number after ``float()`` — neither null nor ``""``
    (``data_type_update.py:37-38`` stores None for both)."""
    import pyarrow.compute as pc
    present = pc.greater(pc.binary_length(arr), 0).fill_null(False)
    return np.asarray(present.to_numpy(zero_copy_only=False), dtype=bool)


def pack_number_cells(cells):
    """:func:`pack_cells` for the number parser: ``str`` cells go through :func:`number_text` first."""
    if cells and isinstance(cells[0], str):
        try:
            arr = number_text(cells)
        except (ImportError, TypeError, ValueError) as _exc:      # mixed str / bytes columns: cell by cell
            cells = [ascii_number_text(c) if isinstance(c, str) else c for c in cells]
        else:
            if not arr.null_count:
                return text_buffers(arr)[:2]
            cells = arr.to_pylist()
    return pack_cells(cells)


def pack_cells(cells):
    """(chars uint8[total], offsets int64[n+1]) of a list of ``str`` / ``bytes`` cells — the layout the GPU parser and
    the byte-wise group-by read.  Arrow does the UTF-8 encoding and the concatenation in C++."""
    n = len(cells)
    if n == 0:
        return np.zeros(1, dtype=np.uint8), np.zeros(1, dtype=np.int64)
    try:
        import pyarrow as pa
        is_text = isinstance(cells[0], str)
        arr = pa.array(cells, type=pa.large_string() if is_text else pa.large_binary())
        if arr.null_count:
            raise ValueError("null cell")
        return text_buffers(arr)[:2]           # a new array: offsets[0] == 0
    except Exception:                          # mixed str / bytes, exotic objects: encode one by one
        enc = [c.encode("utf-8") if isinstance(c, str) else bytes(c) for c in cells]
        offsets = np.zeros(n + 1, dtype=np.int64)
        np.cumsum([len(b) for b in enc], out=offsets[1:])
        return np.frombuffer(b"".join(enc) + b"\0", dtype=np.uint8), offsets


def dictionary_encode(values):
    """Dense codes in first-seen order: (codes uint32, representatives list)."""
    index: dict = {}
    reps = []
    codes = np.empty(len(values), dtype=np.uint32)
    for i, v in enumerate(values):
        k = group_key(v)
        c = index.get(k)
        if c is None:
            c = index[k] = len(reps)
            reps.append(v)
        codes[i] = c
    return codes, reps


def tagged_cell(value) -> bytes:
    """Byte encoding under which two cells are equal exactly when MongoDB's ``$group`` puts them in one group
    (:func:`group_key`): lets ONE byte-wise GPU group-by handle a field that mixes text, numbers and booleans."""
    import struct
    kind = group_key(value)
    if kind[0] == "str":
        return b"s" + value.encode("utf-8")
    if kind[0] == "bool":
        return b"b1" if value else b"b0"
    if kind[0] == "num":
        v = kind[1]
        if v == "nan":
            return b"n" + struct.pack("<Q", 0x7FF8000000000000)
        if v in ("inf", "-inf"):
            return b"n" + struct.pack("<d", float(v))
        if isinstance(v, int):
            if abs(v) <= _EXACT_INT:
                return b"n" + struct.pack("<d", float(v))      # 1 and 1.0 (and -0.0 / 0.0 -> int 0) meet here
            return b"I" + str(v).encode("ascii")               # beyond 2^53: exact decimal text
        return b"n" + struct.pack("<d", v)
    return b"o" + kind[1].encode("utf-8")
