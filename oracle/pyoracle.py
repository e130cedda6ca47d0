"""ctypes binding of the parity oracle (oracle/paimon_oracle.c).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module.  Nothing under paimon_b200/ imports it; the product path has no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import List, Optional, Sequence

import numpy as np

from paimon_b200.columnar import Column, KeyValueBatch
from paimon_b200.merge_function import MergeSpec
from paimon_b200.types import KeyValueSchema, PhysicalType, is_varlen, numpy_dtype

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libpaimon_oracle.so")

SORT_LOSER_TREE, SORT_MIN_HEAP, SORT_BRUTE_FORCE = 0, 1, 2


class _Col(C.Structure):
    _fields_ = [("data", C.c_void_p), ("offsets", C.c_void_p), ("valid", C.c_void_p)]


class _Run(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("cols", C.POINTER(_Col))]


class _Schema(C.Structure):
    _fields_ = [("n_key", C.c_int32), ("n_val", C.c_int32), ("key_types", C.c_void_p),
                ("val_types", C.c_void_p), ("val_nullable", C.c_void_p)]


class _Spec(C.Structure):
    _fields_ = [("engine", C.c_int32), ("sort_engine", C.c_int32), ("ignore_delete", C.c_int32),
                ("remove_record_on_delete", C.c_int32), ("drop_delete", C.c_int32),
                ("n_seq_fields", C.c_int32), ("seq_fields", C.c_void_p), ("seq_ascending", C.c_int32),
                ("agg", C.c_void_p), ("ignore_retract", C.c_void_p),
                ("n_groups", C.c_int32), ("group_seq_start", C.c_void_p),
                ("group_seq_fields", C.c_void_p), ("field_group", C.c_void_p),
                ("group_partial_delete", C.c_void_p), ("bypass_wrapper", C.c_int32),
                ("decimal", C.c_void_p)]


class _OutCol(C.Structure):
    _fields_ = [("data", C.c_void_p), ("offsets", C.c_void_p), ("valid", C.c_void_p),
                ("data_bytes", C.c_int64)]


class _Result(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("n_cols", C.c_int32), ("cols", C.POINTER(_OutCol))]


class OracleError(RuntimeError):
    """The Java path would have thrown (IllegalArgumentException / UnsupportedOperationException)."""


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "paimon_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or (
            os.path.exists(src) and os.path.getmtime(src) > os.path.getmtime(_LIB_PATH)):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.po_merge.restype = C.c_int
        _lib.po_merge.argtypes = [C.POINTER(_Schema), C.POINTER(_Spec), C.c_int32, C.POINTER(_Run),
                                  C.POINTER(C.POINTER(_Result))]
        _lib.po_result_free.argtypes = [C.POINTER(_Result)]
        _lib.po_last_error.restype = C.c_char_p
        _lib.po_merge_order.restype = C.c_int
        _lib.po_merge_order.argtypes = [C.POINTER(_Schema), C.POINTER(_Spec), C.c_int32, C.POINTER(_Run),
                                        C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]
        _lib.po_interval_partition.restype = C.c_int
        _lib.po_interval_partition.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.POINTER(C.c_int32)]
    return _lib


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class _Marshalled:
    """Keeps every numpy buffer alive for the duration of a call."""

    def __init__(self, schema: KeyValueSchema, spec: MergeSpec, runs: Sequence[KeyValueBatch], sort_engine: int,
                 bypass_wrapper: bool = False):
        self.keep: List[np.ndarray] = []
        kt = np.array([int(f.physical) for f in schema.key_type.fields], np.int32)
        vt = np.array([int(f.physical) for f in schema.value_type.fields], np.int32)
        vn = np.array([1 if f.nullable else 0 for f in schema.value_type.fields], np.uint8)
        self.keep += [kt, vt, vn]
        self.schema = _Schema(schema.n_key, schema.n_val, _ptr(kt), _ptr(vt), _ptr(vn))

        sp = spec.normalised(schema.n_val)
        seqf = np.array(sp.seq_fields, np.int32)
        agg = np.array([int(a) for a in sp.agg], np.int32)
        ign = np.array([1 if b else 0 for b in sp.ignore_retract], np.uint8)
        gstart = np.zeros(len(sp.groups) + 1, np.int32)
        gf: List[int] = []
        for i, g in enumerate(sp.groups):
            gf += list(g)
            gstart[i + 1] = len(gf)
        gfields = np.array(gf, np.int32)
        fgroup = np.array(sp.field_group, np.int32)
        gpd = np.array([1 if b else 0 for b in sp.group_partial_delete], np.uint8)
        dec = np.array(sp.decimal, np.int32) if sp.decimal else None
        self.keep += [seqf, agg, ign, gstart, gfields, fgroup, gpd, dec]
        self.spec = _Spec(int(sp.engine), sort_engine, int(sp.ignore_delete), int(sp.remove_record_on_delete),
                          int(sp.drop_delete), len(sp.seq_fields), _ptr(seqf), int(sp.seq_ascending),
                          _ptr(agg), _ptr(ign), len(sp.groups), _ptr(gstart), _ptr(gfields), _ptr(fgroup),
                          _ptr(gpd), int(bypass_wrapper), _ptr(dec))

        self.runs = (_Run * max(1, len(runs)))()
        self.col_arrays = []
        for r, run in enumerate(runs):
            cols = (_Col * schema.n_cols)()
            for ci, col in enumerate(run.columns):
                data = np.ascontiguousarray(col.data)
                offs = None if col.offsets is None else np.ascontiguousarray(col.offsets, dtype=np.int32)
                valid = None if col.valid is None else np.ascontiguousarray(col.valid, dtype=np.uint8)
                self.keep += [a for a in (data, offs, valid) if a is not None]
                cols[ci] = _Col(_ptr(data), _ptr(offs), _ptr(valid))
            self.col_arrays.append(cols)
            self.runs[r] = _Run(run.n_rows, cols)
        self.k = len(runs)


def merge(schema: KeyValueSchema, spec: MergeSpec, runs: Sequence[KeyValueBatch],
          sort_engine: int = SORT_LOSER_TREE, bypass_wrapper: bool = False) -> KeyValueBatch:
    """SortMergeReader over `runs` with the ReducerMergeFunctionWrapper'd merge function of `spec`."""
    m = _Marshalled(schema, spec, runs, sort_engine, bypass_wrapper)
    out = C.POINTER(_Result)()
    rc = lib().po_merge(C.byref(m.schema), C.byref(m.spec), m.k, m.runs, C.byref(out))
    if rc != 0:
        raise OracleError(lib().po_last_error().decode())
    try:
        res = out.contents
        n = res.n_rows
        cols: List[Column] = []
        for ci, t in enumerate(schema.physical_types()):
            oc = res.cols[ci]
            valid = np.ctypeslib.as_array(C.cast(oc.valid, C.POINTER(C.c_uint8)), shape=((n + 7) // 8 + 1,)).copy()
            if is_varlen(t):
                offs = np.ctypeslib.as_array(C.cast(oc.offsets, C.POINTER(C.c_int32)), shape=(n + 1,)).copy()
                nb = int(oc.data_bytes)
                data = (np.ctypeslib.as_array(C.cast(oc.data, C.POINTER(C.c_uint8)), shape=(max(nb, 1),))[:nb].copy()
                        if nb else np.zeros(0, np.uint8))
                cols.append(Column(t, data, offs, valid))
            else:
                dt = np.dtype(numpy_dtype(t))
                raw = np.ctypeslib.as_array(C.cast(oc.data, C.POINTER(C.c_uint8)),
                                            shape=(max(n * dt.itemsize, 1),))[: n * dt.itemsize].copy()
                cols.append(Column(t, raw.view(dt), None, valid))
        return KeyValueBatch(schema, cols)
    finally:
        lib().po_result_free(out)


def merge_order(schema: KeyValueSchema, spec: MergeSpec, runs: Sequence[KeyValueBatch],
                sort_engine: int = SORT_LOSER_TREE):
    """(run,row) pop order of the bare LoserTree / min-heap."""
    m = _Marshalled(schema, spec, runs, sort_engine)
    total = sum(r.n_rows for r in runs)
    out_run = np.zeros(max(total, 1), np.int32)
    out_row = np.zeros(max(total, 1), np.int64)
    n = C.c_int64(0)
    rc = lib().po_merge_order(C.byref(m.schema), C.byref(m.spec), m.k, m.runs, _ptr(out_run), _ptr(out_row),
                              C.byref(n))
    if rc != 0:
        raise OracleError(lib().po_last_error().decode())
    return out_run[: n.value], out_row[: n.value]


def interval_partition(min_keys: Sequence[int], max_keys: Sequence[int]):
    """IntervalPartition over int64 key bounds -> (section_of[file], run_of[file], n_sections)."""
    n = len(min_keys)
    mn = np.array(min_keys, np.int64)
    mx = np.array(max_keys, np.int64)
    sec = np.zeros(max(n, 1), np.int32)
    run = np.zeros(max(n, 1), np.int32)
    ns = C.c_int32(0)
    lib().po_interval_partition(n, _ptr(mn), _ptr(mx), _ptr(sec), _ptr(run), C.byref(ns))
    return sec[:n], run[:n], ns.value


def prepare(schema: KeyValueSchema, spec: MergeSpec, runs: Sequence[KeyValueBatch],
            sort_engine: int = SORT_LOSER_TREE):
    """Marshal once (outside any timed region); see run_prepared."""
    lib()
    return _Marshalled(schema, spec, runs, sort_engine)


def run_prepared(m) -> int:
    """Only the C call (ctypes drops the GIL for its duration): merge and discard, returning the row count.
    Used by bench.py's cpu_baseline so that Python marshalling is not billed to the reference algorithm."""
    out = C.POINTER(_Result)()
    rc = lib().po_merge(C.byref(m.schema), C.byref(m.spec), m.k, m.runs, C.byref(out))
    if rc != 0:
        raise OracleError(lib().po_last_error().decode())
    n = out.contents.n_rows
    lib().po_result_free(out)
    return n
