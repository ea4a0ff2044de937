"""ctypes binding of ``libloexec.so`` (C ABI: ``include/loexec.h``).

The library is loaded from ``learningorchestra_b200/lib/libloexec.so`` (built in-tree by
``learningorchestra_b200.build``).  There is no Python or CPU fallback: if the library is missing
or no H100 is visible, importing this module still works (so CPU-only hosts can run the host-logic
tests) but the first call raises :class:`LoexecError`.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import os

# LOEXEC_LIB overrides the library path (kernel-variant experiments); the default is the in-tree build
LIB_PATH = Path(os.environ.get("LOEXEC_LIB") or Path(__file__).resolve().parent / "lib" / "libloexec.so")

LO_OK = 0
LO_ERR_INVALID = -1
LO_ERR_CUDA = -2
LO_ERR_NOMEM = -3
LO_ERR_NOT_IMPLEMENTED = -4
LO_ERR_NO_DEVICE = -5
LO_ERR_ALIGNMENT = -6

LO_F64, LO_F32, LO_U8, LO_U32 = 1, 2, 3, 4
LO_SYNTH_UNIFORM, LO_SYNTH_EDGES, LO_SYNTH_CONSTCOL, LO_SYNTH_MNIST_U8 = 0, 1, 2, 3
LO_MAX_BINS = 65536
LO_MERGE_AUTO, LO_MERGE_PEER, LO_MERGE_NCCL = 0, 1, 2
LO_GROUP_BCAST = 1
LO_GROUP_INDEPENDENT = 2
LO_GROUP_BLOB_BYTES = 512
LO_GROUP_MAX_DEVICES = 16
LO_GROUP_MAX_COUNTS = 262144
LO_NUM_FLOAT, LO_NUM_INTEGER, LO_NUM_EMPTY, LO_NUM_INVALID, LO_NUM_UNSUPPORTED = 0, 1, 2, 3, 4
LO_FORMAT_MAX_CELL = 310
LO_CSV_OK, LO_CSV_SHORT_ROW, LO_CSV_FIELD_LIMIT, LO_CSV_BAD_UTF8, LO_CSV_NUL, LO_CSV_UNSUPPORTED, LO_CSV_EMPTY = range(7)
LO_CSV_STREAM_WINDOW = 64 << 20
LO_ABI_VERSION = 3

_ERR_NAMES = {
    LO_ERR_INVALID: "LO_ERR_INVALID", LO_ERR_CUDA: "LO_ERR_CUDA", LO_ERR_NOMEM: "LO_ERR_NOMEM",
    LO_ERR_NOT_IMPLEMENTED: "LO_ERR_NOT_IMPLEMENTED", LO_ERR_NO_DEVICE: "LO_ERR_NO_DEVICE",
    LO_ERR_ALIGNMENT: "LO_ERR_ALIGNMENT",
}


class LoexecError(RuntimeError):
    """A libloexec call failed (``code`` is the negative LO_ERR_* value)."""

    def __init__(self, code: int, message: str):
        super().__init__(f"{_ERR_NAMES.get(code, code)}: {message}")
        self.code = code
        self.message = message


class HistSpec(C.Structure):
    _fields_ = [("nbins", C.c_int32), ("flags", C.c_int32),
                ("lo", C.POINTER(C.c_float)), ("hi", C.POINTER(C.c_float))]


class HostTiming(C.Structure):
    _fields_ = [("total_ms", C.c_double), ("h2d_bytes", C.c_double), ("d2h_bytes", C.c_double),
                ("launches", C.c_int64), ("kernel_ms", C.c_double)]


class CsvInfo(C.Structure):
    _fields_ = [("records", C.c_int64), ("ncols", C.c_int64), ("chars", C.c_int64), ("fail_record", C.c_int64),
                ("fail_kind", C.c_int32), ("pad", C.c_int32), ("fail_pos", C.c_int64)]


class CsvWindow(C.Structure):
    _fields_ = [("consumed", C.c_int64), ("records", C.c_int64), ("first_record", C.c_int64), ("ncols", C.c_int64),
                ("chars", C.c_int64), ("peak_device_bytes", C.c_int64), ("done", C.c_int32), ("pad", C.c_int32)]


# every symbol include/loexec.h declares: name -> (restype, argtypes)
_P = C.c_void_p
SIGNATURES = {
    "lo_abi_version": (C.c_int, []),
    "lo_last_error": (C.c_char_p, []),
    "lo_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "lo_init": (C.c_int, [C.c_int, C.POINTER(_P)]),
    "lo_shutdown": (C.c_int, [_P]),
    "lo_ctx_device": (C.c_int, [_P, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_size_t)]),
    "lo_sync": (C.c_int, [_P, _P]),
    "lo_set_tma": (C.c_int, [_P, C.c_int]),
    "lo_launch_count": (C.c_int, [_P, C.POINTER(C.c_int64)]),
    "lo_host_alloc": (C.c_int, [_P, C.c_size_t, C.POINTER(_P)]),
    "lo_host_alloc_flags": (C.c_int, [_P, C.c_size_t, C.c_int32, C.POINTER(_P)]),
    "lo_host_free": (C.c_int, [_P, _P]),
    "lo_table_alloc": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int32, C.POINTER(_P)]),
    "lo_table_wrap": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int32, _P, C.c_int64, C.POINTER(_P)]),
    "lo_table_free": (C.c_int, [_P, _P]),
    "lo_table_info": (C.c_int, [_P, C.POINTER(C.c_int), C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                C.POINTER(C.c_int64), C.POINTER(_P)]),
    "lo_table_upload_col": (C.c_int, [_P, _P, C.c_int32, C.c_int64, _P, C.c_int64]),
    "lo_table_download_col": (C.c_int, [_P, _P, C.c_int32, C.c_int64, _P, C.c_int64, _P]),
    "lo_table_fill_synthetic_dev": (C.c_int, [_P, _P, C.c_int, C.c_uint64, C.c_int64, C.c_double, C.c_double, _P]),
    "lo_table_checksum": (C.c_int, [_P, _P, C.c_int32, C.c_int64, C.POINTER(C.c_uint64)]),
    "lo_selftest_fastdiv": (C.c_int, [_P, C.c_float, C.c_float, C.c_int32, C.POINTER(C.c_int), C.POINTER(C.c_uint64)]),
    "lo_hist_edges": (C.c_int, [C.c_float, C.c_float, C.c_int32, _P]),
    "lo_selftest_edges": (C.c_int, [_P, C.c_float, C.c_float, C.c_int32, C.POINTER(C.c_int), C.POINTER(C.c_uint64)]),
    "lo_edge_tables_info": (C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(C.c_int64)]),
    "lo_minmax_cast_dev": (C.c_int, [_P, _P, C.POINTER(C.c_int32), C.c_int32, _P, _P]),
    "lo_minmax_decode": (C.c_int, [_P, C.c_int32, _P, _P, _P]),
    "lo_project_cast_dev": (C.c_int, [_P, _P, C.POINTER(C.c_int32), C.c_int32, _P, _P]),
    "lo_project_cast_hist_dev": (C.c_int, [_P, _P, C.POINTER(C.c_int32), C.c_int32, _P, C.POINTER(HistSpec), _P, _P]),
    "lo_hist_u8_cols_dev": (C.c_int, [_P, _P, C.POINTER(C.c_int32), C.c_int32, _P, _P]),
    "lo_counts_alloc": (C.c_int, [_P, C.c_int64, C.POINTER(_P)]),
    "lo_counts_free": (C.c_int, [_P, _P]),
    "lo_counts_zero_dev": (C.c_int, [_P, _P, C.c_int64, _P]),
    "lo_counts_download": (C.c_int, [_P, _P, C.c_int64, _P, _P]),
    "lo_project_cast_hist_host": (C.c_int, [_P, C.POINTER(_P), C.c_int64, C.c_int32, C.POINTER(_P),
                                            C.POINTER(HistSpec), _P, C.POINTER(HostTiming)]),
    "lo_hist_u8_cols_host": (C.c_int, [_P, C.POINTER(_P), C.c_int64, C.c_int32, _P, C.POINTER(HostTiming)]),
    "lo_group_create_local": (C.c_int, [C.POINTER(_P), C.c_int32, C.c_int32, C.POINTER(_P)]),
    "lo_group_rank_begin": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P), _P]),
    "lo_group_rank_connect": (C.c_int, [_P, _P]),
    "lo_group_destroy": (C.c_int, [_P]),
    "lo_group_info": (C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "lo_group_shard": (C.c_int, [_P, C.c_int64, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "lo_group_project_cast_hist_dev": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_int32), C.c_int32, C.POINTER(_P),
                                                 C.POINTER(HistSpec), C.c_int32, C.POINTER(_P)]),
    "lo_group_hist_u8_cols_dev": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.POINTER(_P)]),
    "lo_group_minmax_cast_dev": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_int32), C.c_int32, C.POINTER(_P)]),
    "lo_group_project_cast_hist_host": (C.c_int, [_P, C.POINTER(_P), C.c_int64, C.c_int32, C.POINTER(_P),
                                                  C.POINTER(HistSpec), _P, C.c_int32, C.POINTER(HostTiming)]),
    "lo_group_hist_u8_cols_host": (C.c_int, [_P, C.POINTER(_P), C.c_int64, C.c_int32, _P, C.c_int32, C.POINTER(HostTiming)]),
    "lo_group_result": (C.c_int, [_P, C.c_int32, C.c_int64, _P]),
    "lo_group_result_dev": (C.c_int, [_P, C.c_int32, C.POINTER(_P)]),
    "lo_group_barrier_dev": (C.c_int, [_P, C.POINTER(_P)]),
    "lo_group_timeouts": (C.c_int, [_P, C.POINTER(C.c_uint64)]),
    "lo_ctx_bind_numa": (C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "lo_value_counts_u32_host": (C.c_int, [_P, _P, C.c_int64, C.c_uint32, _P, C.POINTER(HostTiming)]),
    "lo_value_counts_f64_host": (C.c_int, [_P, _P, C.c_int64, _P, _P, C.c_int64, C.POINTER(C.c_int64), C.POINTER(HostTiming)]),
    "lo_value_counts_str_host": (C.c_int, [_P, _P, _P, C.c_int64, _P, _P, C.c_int64, C.POINTER(C.c_int64), C.POINTER(HostTiming)]),
    "lo_parse_number_host": (C.c_int, [_P, _P, _P, C.c_int64, _P, _P, C.POINTER(HostTiming)]),
    "lo_format_number_host": (C.c_int, [_P, _P, _P, C.c_int64, _P, _P, C.c_int64, C.POINTER(HostTiming)]),
    "lo_minmax_cast_host": (C.c_int, [_P, C.POINTER(_P), C.c_int64, C.c_int32, _P, _P, _P, C.POINTER(HostTiming)]),
    "lo_csv_read_host": (C.c_int, [_P, _P, C.c_int64, C.POINTER(_P), C.POINTER(CsvInfo), C.POINTER(HostTiming)]),
    "lo_csv_columns_host": (C.c_int, [_P, _P, _P, C.c_int64, C.POINTER(HostTiming)]),
    "lo_csv_free": (C.c_int, [_P]),
    "lo_csv_stream_open": (C.c_int, [_P, C.c_int64, C.POINTER(_P)]),
    "lo_csv_stream_push": (C.c_int, [_P, _P, C.c_int64, C.c_int32, C.POINTER(CsvWindow), C.POINTER(CsvInfo),
                                     C.POINTER(HostTiming)]),
    "lo_csv_stream_columns": (C.c_int, [_P, _P, _P, C.c_int64, C.POINTER(HostTiming)]),
    "lo_csv_stream_free": (C.c_int, [_P]),
}

_lib = None


def load() -> C.CDLL:
    """Load libloexec.so and bind every declared symbol; raises LoexecError if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise LoexecError(LO_ERR_NO_DEVICE,
                          f"{LIB_PATH} is missing — build it with `python -m learningorchestra_b200.build` "
                          "(__graft_entry__.build()); there is no CPU fallback")
    lib = C.CDLL(str(LIB_PATH))
    lax = bool(os.environ.get("LOEXEC_LAX"))          # A/B measurements against an older build (scripts/ab_libs.py)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name, None) if lax else getattr(lib, name)   # AttributeError = header / library mismatch
        if fn is None:
            continue
        fn.restype = res
        fn.argtypes = args
    if lib.lo_abi_version() != LO_ABI_VERSION and not lax:
        raise LoexecError(LO_ERR_INVALID, f"ABI version {lib.lo_abi_version()} != {LO_ABI_VERSION}")
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != LO_OK:
        msg = load().lo_last_error()
        raise LoexecError(rc, msg.decode("utf-8", "replace") if msg else "")
