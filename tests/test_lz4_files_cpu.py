"""LZ4 files on the host, without a GPU: the ORC host build (tests/native/orc_lz4_host_check.cc over orc_meta.cc +
lz4_device.cuh + orc_device.cuh, the sources the device path compiles) decodes pyarrow.orc files written with compression="lz4" (CompressionKind 4: one raw LZ4 block
per compression chunk, the footers too) of every KeyValue type at several compression block sizes, equal to pyarrow;
and pg_parquet_open accepts Parquet codec 5 (Hadoop-framed LZ4) files with pyarrow's counts, while codec 7 (LZ4_RAW)
stays refused."""
import ctypes as C
import io
import os
import struct
import subprocess

import numpy as np
import pyarrow.parquet as pq
import pytest

import orc_util
import parquet_pages as P
from lz4_parquet import read_struct, to_hadoop_lz4
from paimon_b200 import _native as N
from paimon_b200 import datagen
from test_orc_cpu import _check, _table
from test_parquet_cpu import _schema_handle

from parquet_util import write_kv_parquet


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    """orc_util.build's library, from the harness that also decodes LZ4 chunks"""
    so = str(tmp_path_factory.mktemp("orc_lz4") / "liborc_lz4_host.so")
    csrc = os.path.join(orc_util.ROOT, "paimon_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + csrc, "-o", so,
                           os.path.join(orc_util.ROOT, "tests", "native", "orc_lz4_host_check.cc"),
                           os.path.join(csrc, "orc_meta.cc")])
    lib = C.CDLL(so)
    lib.orc_host_decode.restype = C.c_void_p
    lib.orc_host_decode.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p]
    lib.orc_host_error.restype = C.c_char_p
    lib.orc_host_rows.restype = C.c_longlong
    lib.orc_host_rows.argtypes = [C.c_void_p]
    lib.orc_host_data.restype = C.c_void_p
    lib.orc_host_data.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_longlong)]
    lib.orc_host_offsets.restype = C.c_void_p
    lib.orc_host_offsets.argtypes = [C.c_void_p, C.c_int]
    lib.orc_host_validity.restype = C.c_void_p
    lib.orc_host_validity.argtypes = [C.c_void_p, C.c_int]
    lib.orc_host_free.argtypes = [C.c_void_p]
    return lib


@pytest.mark.parametrize("opts", [
    dict(compression="lz4"),
    dict(compression="lz4", compression_block_size=128 * 1024, stripe_size=64 * 1024),     # many stripes
    dict(compression="lz4", compression_block_size=256 * 1024),
    dict(compression="lz4", compression_block_size=1024 * 1024),
    dict(compression="lz4", file_version="0.11", dictionary_key_size_threshold=1.0),
])
def test_orc_lz4_against_pyarrow(lib, tmp_path, opts):
    for n, null_p in ((0, 0.0), (1, 0.0), (31, 0.3), (5000, 0.25), (40000, 0.0), (20000, 0.9)):
        _check(lib, _table(n, seed=n + 1, null_p=null_p), str(tmp_path / "t.orc"), **opts)


def _open(sh, blob):
    lib = N.load()
    buf = np.frombuffer(blob, np.uint8)
    h = C.c_uint64(0)
    return lib.pg_parquet_open(sh, buf.ctypes.data, len(buf), C.byref(h)), h.value


@pytest.mark.parametrize("opts", [dict(), dict(use_dictionary=False), dict(data_page_version="2.0"),
                                  dict(row_group_size=1000, data_page_size=2048)])
def test_parquet_open_accepts_codec_5(tmp_path, opts):
    schema = datagen.schema_c3(n_i64=2, n_f64=2, n_str=2)
    run = datagen.make_runs(schema, 1, 5000, seed=4, null_prob=0.3)[0]
    path = str(tmp_path / "plain.parquet")
    write_kv_parquet(run, path, **opts)
    blob = to_hadoop_lz4(open(path, "rb").read())
    lib = N.load()
    sh = _schema_handle(schema)
    st, h = _open(sh, blob)
    assert st == 0, lib.pg_last_error()
    info = N.PgParquetInfo()
    assert lib.pg_parquet_describe(h, C.byref(info)) == 0
    md = pq.ParquetFile(io.BytesIO(blob)).metadata
    (flen,) = struct.unpack("<I", blob[-8:-4])
    footer, _ = read_struct(blob, len(blob) - 8 - flen)
    assert {cc[3][1][4][1] for rg in footer[4][1][1] for cc in rg[1][1][1]} == {5}
    assert info.n_rows == md.num_rows == run.n_rows
    assert info.n_row_groups == md.num_row_groups
    assert info.n_columns == md.num_columns == schema.n_cols
    n_dict = sum(1 for g in range(md.num_row_groups) for c in range(md.num_columns)
                 if md.row_group(g).column(c).has_dictionary_page)
    assert info.n_dictionary_pages == n_dict
    assert info.n_data_pages >= md.num_row_groups * md.num_columns
    assert pq.read_table(io.BytesIO(blob)).equals(pq.read_table(path))     # Arrow's Hadoop-LZ4 reader agrees
    assert lib.pg_parquet_free(h) == 0
    assert lib.pg_schema_free(sh) == 0


def test_parquet_open_keeps_refusing_lz4_raw(tmp_path):
    schema = datagen.schema_c1()
    run = datagen.make_runs(schema, 1, 100, seed=1)[0]
    p = str(tmp_path / "raw.parquet")
    write_kv_parquet(run, p, compression="lz4")                              # pyarrow writes codec 7
    sh = _schema_handle(schema)
    st, _ = _open(sh, open(p, "rb").read())
    assert st == 2 and b"compression codec 7" in N.load().pg_last_error()


def test_page_builder_lz4_pages_read_by_pyarrow():
    """The builder's headers case (CRCs, statistics, unknown header fields, an index page) made codec 5, its first V2
    page stored uncompressed: pyarrow reads it to the builder's values, with the recomputed CRCs verified."""
    case = P.headers_case(P.UNCOMPRESSED)
    blob = to_hadoop_lz4(case.files[0], raw_first_v2=True)
    t = pq.read_table(io.BytesIO(blob), page_checksum_verification=True)
    assert P.arrow_values(t.column("v"), "STRING") == case.expected
