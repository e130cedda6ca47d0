"""CPU-side checks of the Parquet host parser (Thrift footer + page headers) against pyarrow's metadata."""
import ctypes as C
import os

import numpy as np
import pyarrow.parquet as pq
import pytest

import parquet_pages as P
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.sort_merge_reader import _SchemaHandle
from paimon_b200.types import DataField, KeyValueSchema, RowType

from parquet_util import write_kv_parquet

PG_ERR_UNSUPPORTED, PG_ERR_FORMAT = 2, 6


def _open(schema_handle, path):
    lib = N.load()
    buf = np.fromfile(path, dtype=np.uint8)
    h = C.c_uint64(0)
    st = lib.pg_parquet_open(schema_handle, buf.ctypes.data, len(buf), C.byref(h))
    return st, h.value, buf


def _schema_handle(schema):
    """pg_schema_create needs no device."""
    lib = N.load()
    kf = (N.PgField * schema.n_key)(*[N.PgField(int(f.physical), 0) for f in schema.key_type.fields])
    vf = (N.PgField * schema.n_val)(*[N.PgField(int(f.physical), int(f.nullable)) for f in schema.value_type.fields])
    desc = N.PgSchemaDesc(schema.n_key, schema.n_val, kf, vf)
    h = C.c_uint64(0)
    assert lib.pg_schema_create(C.byref(desc), C.byref(h)) == 0
    return h.value


@pytest.mark.parametrize("opts", [dict(), dict(use_dictionary=False), dict(data_page_version="2.0"),
                                  dict(row_group_size=1000, data_page_size=2048)])
def test_footer_and_page_walk_match_pyarrow(tmp_path, opts):
    schema = datagen.schema_c3(n_i64=2, n_f64=2, n_str=2)
    run = datagen.make_runs(schema, 1, 5000, seed=4, null_prob=0.3)[0]
    path = str(tmp_path / "data.parquet")
    write_kv_parquet(run, path, **opts)
    sh = _schema_handle(schema)
    st, h, _ = _open(sh, path)
    lib = N.load()
    assert st == 0, lib.pg_last_error()
    info = N.PgParquetInfo()
    assert lib.pg_parquet_describe(h, C.byref(info)) == 0
    md = pq.ParquetFile(path).metadata
    assert info.n_rows == md.num_rows == run.n_rows
    assert info.n_row_groups == md.num_row_groups
    assert info.n_columns == md.num_columns == schema.n_cols
    n_dict = sum(1 for g in range(md.num_row_groups) for c in range(md.num_columns)
                 if md.row_group(g).column(c).has_dictionary_page)
    assert info.n_dictionary_pages == n_dict
    assert info.n_data_pages >= md.num_row_groups * md.num_columns
    assert lib.pg_parquet_free(h) == 0
    assert lib.pg_schema_free(sh) == 0


def test_unsupported_files_are_refused(tmp_path):
    schema = datagen.schema_c1()
    run = datagen.make_runs(schema, 1, 100, seed=1)[0]
    lib = N.load()
    sh = _schema_handle(schema)
    p = str(tmp_path / "z.parquet")
    write_kv_parquet(run, p, compression="lz4")
    st, _, _ = _open(sh, p)
    assert st == 2 and b"compression codec" in lib.pg_last_error()         # PG_ERR_UNSUPPORTED
    p = str(tmp_path / "zstd.parquet")                  # Paimon's default codec is accepted
    write_kv_parquet(run, p, compression="zstd")
    st, h_z, _ = _open(sh, p)
    assert st == 0
    lib.pg_parquet_free(h_z)
    p = str(tmp_path / "delta.parquet")                 # DELTA_BINARY_PACKED integers are accepted ...
    write_kv_parquet(run, p, use_dictionary=False, column_encoding="DELTA_BINARY_PACKED")
    st, h_ok, _ = _open(sh, p)
    assert st == 0
    lib.pg_parquet_free(h_ok)
    p = str(tmp_path / "bss.parquet")                   # ... BYTE_STREAM_SPLIT is not
    write_kv_parquet(run, p, use_dictionary=False, column_encoding="BYTE_STREAM_SPLIT")
    st, _, _ = _open(sh, p)
    assert st == 2 and b"encoding" in lib.pg_last_error()
    junk = np.frombuffer(b"not a parquet file at all.....", dtype=np.uint8)
    h = C.c_uint64(0)
    assert lib.pg_parquet_open(sh, junk.ctypes.data, len(junk), C.byref(h)) == 6   # PG_ERR_FORMAT
    other = datagen.schema_c2()
    sh2 = _schema_handle(other)
    p = str(tmp_path / "c1.parquet")
    write_kv_parquet(run, p)
    st, _, _ = _open(sh2, p)
    assert st == 2                                                           # column count mismatch


def _open_pages_file(data, vtype):
    """pg_parquet_open's status on a parquet_pages.kv_file (the handles it made are freed)"""
    lib = N.load()
    sh = _schema_handle(KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("v", vtype, True))), ["pk"]))
    buf = np.frombuffer(data, np.uint8)
    h = C.c_uint64(0)
    st = lib.pg_parquet_open(sh, buf.ctypes.data, len(buf), C.byref(h))
    if st == 0:
        assert lib.pg_parquet_free(h.value) == 0
    assert lib.pg_schema_free(sh) == 0
    return st


def test_open_refuses_what_the_device_page_walk_refuses():
    """pg_parquet_open runs the page walk of the device decoder on the host.  Of the malformed files, the one whose
    dictionary page claims more entries than its body holds is refused there; the others break value streams, which
    only the decode reads.  A dictionary page between two data pages is refused as an encoding the decoder lacks."""
    statuses = {name: _open_pages_file(*make()) for name, make in P.malformed_cases().items()}
    assert {k: v for k, v in statuses.items() if v != 0} == {"dict_page_overclaims": PG_ERR_FORMAT}
    page = lambda vals: P.data_page_v1(len(vals), P.plain(P.INT64, vals), P.E_PLAIN, defs=P.levels([True] * len(vals)))
    pages = [page(list(range(50))), P.dictionary_page(4, P.plain(P.INT64, [1, 2, 3, 4])), page(list(range(50, 100)))]
    data = P.kv_file([100], [P.ValueColumn("v", P.INT64, True, [pages])])
    assert _open_pages_file(data, "BIGINT") == PG_ERR_UNSUPPORTED
    assert b"encoding" in N.load().pg_last_error()


def test_decode_without_device_fails_loudly(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    schema = datagen.schema_c1()
    run = datagen.make_runs(schema, 1, 100, seed=1)[0]
    p = str(tmp_path / "a.parquet")
    write_kv_parquet(run, p)
    sh = _schema_handle(schema)
    st, h, _ = _open(sh, p)
    assert st == 0
    out = C.c_uint64(0)
    assert N.load().pg_parquet_read_run(h, C.byref(out)) != 0
