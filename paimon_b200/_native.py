"""ctypes binding of libpaimon_gpu.so (include/paimon_gpu.h).

This is the Python stand-in for the JNI shim (jni/paimon_gpu_jni.cc): one thin wrapper per C-ABI
function, opaque integer handles, errors raised from ``pg_last_error``.  The library is the only
implementation of the path: if it is missing or no CUDA device is present, importing / initialising
fails loudly — there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
# PAIMON_GPU_LIB: another build of the same library (kernel A/B experiments; profiles/README.md)
LIB_PATH = os.environ.get("PAIMON_GPU_LIB") or os.path.join(_HERE, "libpaimon_gpu.so")

PG_MEM_HOST, PG_MEM_DEVICE = 0, 1


class PgField(C.Structure):
    _fields_ = [("type", C.c_int32), ("nullable", C.c_int32)]


class PgSchemaDesc(C.Structure):
    _fields_ = [("n_key", C.c_int32), ("n_val", C.c_int32),
                ("key_fields", C.POINTER(PgField)), ("val_fields", C.POINTER(PgField))]


class PgMergeSpec(C.Structure):
    _fields_ = [("engine", C.c_int32), ("ignore_delete", C.c_int32), ("remove_record_on_delete", C.c_int32),
                ("drop_delete", C.c_int32), ("n_seq_fields", C.c_int32), ("seq_fields", C.c_void_p),
                ("seq_ascending", C.c_int32), ("agg", C.c_void_p), ("ignore_retract", C.c_void_p),
                ("n_sequence_groups", C.c_int32), ("group_seq_start", C.c_void_p),
                ("group_seq_fields", C.c_void_p), ("field_group", C.c_void_p),
                ("group_partial_delete", C.c_void_p), ("read_fields", C.c_void_p), ("decimal", C.c_void_p)]


class PgColumn(C.Structure):
    _fields_ = [("data", C.c_void_p), ("offsets", C.c_void_p), ("validity", C.c_void_p)]


class PgRunDesc(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("cols", C.POINTER(PgColumn))]


class PgOutColumn(C.Structure):
    _fields_ = [("data", C.c_void_p), ("offsets", C.c_void_p), ("validity", C.c_void_p),
                ("data_bytes", C.c_int64)]


class PgBatch(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("n_cols", C.c_int32), ("cols", C.POINTER(PgOutColumn))]


class PgStats(C.Structure):
    _fields_ = [("rows_in", C.c_int64), ("rows_out", C.c_int64), ("bytes_h2d", C.c_int64),
                ("bytes_d2h", C.c_int64), ("bytes_out", C.c_int64), ("n_tiles", C.c_int32),
                ("n_levels", C.c_int32), ("ms_partition", C.c_float), ("ms_plan", C.c_float),
                ("ms_alloc", C.c_float), ("ms_emit", C.c_float), ("ms_total", C.c_float), ("launches", C.c_int32)]


class PgParquetInfo(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("n_row_groups", C.c_int32), ("n_columns", C.c_int32),
                ("n_data_pages", C.c_int32), ("n_dictionary_pages", C.c_int32), ("ms_decode", C.c_float),
                ("launches", C.c_int32)]


class PgFileDesc(C.Structure):
    _fields_ = [("bytes", C.c_void_p), ("size", C.c_int64), ("mem", C.c_int32), ("run", C.c_int32)]


class PgSectionInfo(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("file_bytes", C.c_int64), ("page_bytes", C.c_int64),
                ("decoded_bytes", C.c_int64), ("n_files", C.c_int32), ("n_runs", C.c_int32), ("n_chunks", C.c_int32),
                ("n_data_pages", C.c_int32), ("n_dictionary_pages", C.c_int32), ("launches", C.c_int32),
                ("ms_decode", C.c_float)]


class PgParquetWriteOptions(C.Structure):
    _fields_ = [("row_group_rows", C.c_int64), ("page_rows", C.c_int64)]


class PgFileMeta(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("file_bytes", C.c_int64), ("min_sequence_number", C.c_int64),
                ("max_sequence_number", C.c_int64), ("delete_row_count", C.c_int64), ("n_row_groups", C.c_int32),
                ("n_pages", C.c_int32), ("ms_encode", C.c_float), ("launches", C.c_int32)]


class PaimonGpuError(RuntimeError):
    """A non-zero pg_status.  `.status` holds the code (PG_ERR_*)."""

    def __init__(self, status: int, message: str):
        super().__init__(f"[pg_status {status}] {message}")
        self.status = status
        self.message = message


class UnsupportedOnDevice(PaimonGpuError):
    """PG_ERR_UNSUPPORTED: the spec is refused at plan time (no CPU fallback)."""


class MergeFunctionError(PaimonGpuError):
    """PG_ERR_MERGE_FUNCTION: the reference MergeFunction would have thrown."""


_SIGNATURES = {
    "pg_last_error": (C.c_char_p, []),
    "pg_abi_version": (C.c_int32, []),
    "pg_init": (C.c_int32, [C.c_int32]),
    "pg_shutdown": (C.c_int32, []),
    "pg_schema_create": (C.c_int32, [C.POINTER(PgSchemaDesc), C.POINTER(C.c_uint64)]),
    "pg_schema_free": (C.c_int32, [C.c_uint64]),
    "pg_schema_info": (C.c_int32, [C.c_uint64, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "pg_merge_spec_create": (C.c_int32, [C.c_uint64, C.POINTER(PgMergeSpec), C.POINTER(C.c_uint64)]),
    "pg_merge_spec_free": (C.c_int32, [C.c_uint64]),
    "pg_run_open": (C.c_int32, [C.c_uint64, C.POINTER(PgRunDesc), C.c_int32, C.POINTER(C.c_uint64)]),
    "pg_run_free": (C.c_int32, [C.c_uint64]),
    "pg_merge_open": (C.c_int32, [C.c_uint64, C.POINTER(C.c_uint64), C.c_int32, C.POINTER(C.c_uint64)]),
    "pg_merge_rebind": (C.c_int32, [C.c_uint64, C.POINTER(C.c_uint64), C.c_int32, C.c_void_p]),
    "pg_trim": (C.c_int32, []),
    "pg_merge_execute": (C.c_int32, [C.c_uint64]),
    "pg_merge_device_batch": (C.c_int32, [C.c_uint64, C.POINTER(PgBatch)]),
    "pg_merge_fetch": (C.c_int32, [C.c_uint64, C.POINTER(PgOutColumn), C.c_int32]),
    "pg_merge_release": (C.c_int32, [C.c_uint64]),
    "pg_merge_stats": (C.c_int32, [C.c_uint64, C.POINTER(PgStats)]),
    "pg_merge_stream": (C.c_int32, [C.c_uint64, C.POINTER(C.c_void_p)]),
    "pg_merge_free": (C.c_int32, [C.c_uint64]),
    "pg_interval_partition": (C.c_int32, [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.POINTER(C.c_int32)]),
    "pg_run_layout": (C.c_int32, [C.c_uint64, C.POINTER(C.c_int64), C.c_void_p, C.c_void_p, C.c_int32]),
    "pg_run_fetch": (C.c_int32, [C.c_uint64, C.POINTER(PgOutColumn), C.c_int32]),
    "pg_run_slice": (C.c_int32, [C.c_uint64, C.c_int64, C.c_int64, C.POINTER(C.c_uint64), C.POINTER(C.c_int64)]),
    "pg_thread_stream": (C.c_int32, [C.POINTER(C.c_void_p)]),
    "pg_files_upload_begin": (C.c_int32, [C.POINTER(PgFileDesc), C.c_int32, C.POINTER(C.c_uint64)]),
    "pg_files_upload_wait": (C.c_int32, [C.c_uint64, C.POINTER(PgFileDesc), C.c_int32]),
    "pg_files_upload_free": (C.c_int32, [C.c_uint64]),
    "pg_export_arrow": (C.c_int32, [C.c_uint64, C.POINTER(C.c_char_p), C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "pg_parquet_open": (C.c_int32, [C.c_uint64, C.c_void_p, C.c_int64, C.POINTER(C.c_uint64)]),
    "pg_parquet_describe": (C.c_int32, [C.c_uint64, C.POINTER(PgParquetInfo)]),
    "pg_parquet_read_run": (C.c_int32, [C.c_uint64, C.POINTER(C.c_uint64)]),
    "pg_parquet_free": (C.c_int32, [C.c_uint64]),
    "pg_parquet_read_section": (C.c_int32, [C.c_uint64, C.POINTER(PgFileDesc), C.c_int32, C.c_int32,
                                            C.POINTER(C.c_char_p), C.c_void_p, C.POINTER(C.c_uint64),
                                            C.POINTER(PgSectionInfo)]),
    "pg_orc_read_section": (C.c_int32, [C.c_uint64, C.POINTER(PgFileDesc), C.c_int32, C.c_int32,
                                        C.POINTER(C.c_char_p), C.c_void_p, C.POINTER(C.c_uint64),
                                        C.POINTER(PgSectionInfo)]),
    "pg_parquet_file_device_image": (C.c_int32, [C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    "pg_run_apply_deletion_vector": (C.c_int32, [C.c_uint64, C.c_void_p, C.c_int64, C.POINTER(C.c_uint64)]),
    "pg_parquet_encode": (C.c_int32, [C.c_uint64, C.POINTER(C.c_char_p), C.c_int64, C.c_int64,
                                      C.POINTER(PgParquetWriteOptions), C.POINTER(C.c_uint64)]),
    "pg_parquet_file_meta": (C.c_int32, [C.c_uint64, C.POINTER(PgFileMeta)]),
    "pg_parquet_file_column_stats": (C.c_int32, [C.c_uint64, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                                 C.c_void_p, C.c_void_p]),
    "pg_parquet_file_fetch": (C.c_int32, [C.c_uint64, C.c_void_p, C.c_int64]),
    "pg_parquet_file_free": (C.c_int32, [C.c_uint64]),
}

_lib: Optional[C.CDLL] = None
_initialised_device: Optional[int] = None


def exported_symbols():
    return sorted(_SIGNATURES)


def load() -> C.CDLL:
    """dlopen the library (no CUDA call yet).  Fails loudly when the extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `make` (or __graft_entry__.build()). "
                "paimon_b200 has no CPU fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(status: int) -> None:
    if status != 0:
        msg = load().pg_last_error().decode(errors="replace")
        if status == 2:
            raise UnsupportedOnDevice(status, msg)
        if status == 4:
            raise MergeFunctionError(status, msg)
        raise PaimonGpuError(status, msg)


def init(device: int = 0) -> C.CDLL:
    """pg_init on `device`; raises PaimonGpuError when there is no CUDA device."""
    global _initialised_device
    lib = load()
    if _initialised_device != device:
        check(lib.pg_init(device))
        _initialised_device = device
    return lib
