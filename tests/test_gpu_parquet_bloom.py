"""Parquet bloom filters of the files the device encoder writes (pg_parquet_encode_bloom), against the independent model
(tests/parquet_bloom_reference.py): every filter equals the model's over its chunk's rows bit for bit, each bitset
starts on a 32-byte boundary, every non-NULL value is found in its chunk's filter, the filters sit between the page
index (or the last page) and the footer, and pyarrow and the device's own decoder read the file as they read the file
without filters.  Uncompressed and zstd, with and without the page index.  Needs an H100."""
import ctypes as C
import os
import random

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import parquet_bloom_reference as R
import stats_reference as S
from paimon_b200 import _native as N
from paimon_b200.columnar import KeyValueBatch
from paimon_b200.compact_rewriter import MergeTreeCompactRewriter, file_column_names
from paimon_b200.format import read_section
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.merge_tree_readers import DataFileMeta, IntervalPartition
from paimon_b200.sort_merge_reader import SortedRunReader, _SchemaHandle
from paimon_b200.types import PhysicalType

from parquet_util import arrow_to_batch, write_kv_parquet
from test_gpu_parquet_write import all_types_schema, random_rows

pytestmark = pytest.mark.gpu

SMALL = dict(page_rows=64, row_group_rows=256)
BOOL_COL = 11                    # all_types_schema's file column 'b'


def encode(schema, batch, codec, bloom, page_index=0, row0=0, n=-1, page_rows=0, row_group_rows=0,
           device_image=False, level=1, raw_bloom=None):
    """-> file bytes of pg_parquet_encode_bloom with `bloom` [(file column, ndv, fpp)] (None: a NULL options
    pointer), or of pg_parquet_encode_compressed when bloom is 'compressed'; with device_image also the device decoder's
    batch of the file's device image."""
    lib = N.init(0)
    sh = _SchemaHandle(schema, 0)
    rd = SortedRunReader(schema, batch)
    names = file_column_names(schema)
    arr = (C.c_char_p * len(names))(*[x.encode() for x in names])
    opts = N.PgParquetWriteOptions(row_group_rows, page_rows, page_index)
    fh = C.c_uint64(0)
    try:
        h = rd._open(sh.handle)
        if bloom == "compressed":
            N.check(lib.pg_parquet_encode_compressed(h, arr, row0, n, C.byref(opts), codec, level, C.byref(fh)))
        else:
            if raw_bloom is not None:
                b = raw_bloom
            elif bloom is None:
                b = None
            else:
                cols = (N.PgParquetBloomColumn * max(len(bloom), 1))(*[N.PgParquetBloomColumn(*x) for x in bloom])
                b = N.PgParquetBloomOptions(len(bloom), cols)
            N.check(lib.pg_parquet_encode_bloom(h, arr, row0, n, C.byref(opts), codec, level,
                                                C.byref(b) if b is not None else None, C.byref(fh)))
        try:
            meta = N.PgFileMeta()
            N.check(lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
            buf = np.zeros(max(meta.file_bytes, 1), np.uint8)
            N.check(lib.pg_parquet_file_fetch(fh.value, buf.ctypes.data, meta.file_bytes))
            out = bytes(buf[: meta.file_bytes])
            if not device_image:
                return out
            ptr, size = C.c_void_p(0), C.c_int64(0)
            N.check(lib.pg_parquet_file_device_image(fh.value, C.byref(ptr), C.byref(size)))
            assert size.value == len(out)
            readers, _ = read_section(schema, [((ptr.value, size.value), 0)], 1)
            try:
                return out, readers[0].read_batch()
            finally:
                for r in readers:
                    r.close()
        finally:
            lib.pg_parquet_file_free(fh.value)
    finally:
        rd.close()
        sh.close()


def footer_start(data):
    return len(data) - 8 - int.from_bytes(data[-8:-4], "little")


def check_filters(data, batch, bloom, row0=0, n=-1, **writer_args):
    """Holds every filter of `data` to the model; returns the file offset of the first filter."""
    want = R.file_bitsets(batch, bloom, row0, n, **writer_args)
    got = R.file_filters(data)
    assert len(got) == len(want)
    size = {c: R.num_bytes(ndv, fpp) for c, ndv, fpp in bloom}
    if n < 0:
        n = batch.n_rows - row0
    groups = S.row_groups(n, **writer_args)
    offsets = []
    for g, (grow, wrow) in enumerate(zip(got, want)):
        for c, (f, w) in enumerate(zip(grow, wrow)):
            where = f"row group {g} column {c}"
            assert (f is None) == (w is None), where
            if f is None:
                continue
            assert f["header"][1] == size[c] and f["bitset_offset"] % 32 == 0, where
            assert f["length"] == f["bitset_offset"] - f["offset"] + size[c], where
            assert f["bitset"] == w, where
            # every non-NULL value of the chunk is found
            a, b = groups[g]
            bits = np.frombuffer(f["bitset"], "<u4")
            assert all(R.find(bits, int(h)) for h in R.column_hashes(batch.columns[c], row0 + a, row0 + b)), where
            offsets.append((f["offset"], f["bitset_offset"] + size[c]))
    if not offsets:
        return footer_start(data)
    # row group major, then column, each one behind the last (a gap below 32 bytes before each header), the footer
    # right behind the last
    assert offsets == sorted(offsets)
    assert all(0 <= b[0] - a[1] < 32 for a, b in zip(offsets, offsets[1:]))
    assert offsets[-1][1] == footer_start(data)
    return offsets[0][0]


def check_against_plain(schema, batch, codec, bloom, page_index=0, row0=0, n=-1, **writer_args):
    on = encode(schema, batch, codec, bloom, page_index, row0, n, **writer_args)
    off = encode(schema, batch, codec, "compressed", page_index, row0, n, **writer_args)
    first = check_filters(on, batch, bloom, row0, n, **writer_args)
    end = footer_start(off)
    assert first - end < 32 and on[:end] == off[:end] and not any(on[end:first])
    assert all(f is None for row in R.file_filters(off) for f in row)
    # (repr: NaN equals NaN, -0.0 differs from +0.0)
    assert repr(pq.read_table(pa.BufferReader(on)).to_pydict()) == repr(pq.read_table(pa.BufferReader(off)).to_pydict())
    return on


def all_but_bool(schema, ndv=0, fpp=0.01):
    return [(c, ndv, fpp) for c, t in enumerate(schema.physical_types()) if t != PhysicalType.BOOL]


def mixed_sizes(schema):
    """1 MiB filters (no ndv), 2 KiB (1000 at 0.01), and a 32-byte one that nearly every value saturates"""
    cycle = [(0, 0.01), (1000, 0.01), (10, 0.1), (100000, 0.05)]
    return [(c,) + cycle[i % len(cycle)] for i, (c, _, _) in enumerate(all_but_bool(schema))]


@pytest.mark.parametrize("codec", [0, 6])
@pytest.mark.parametrize("page_index", [0, 1])
@pytest.mark.parametrize("null_p", [0.0, 0.3, 1.0])
def test_all_types(codec, page_index, null_p):
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(int(10 * null_p) + page_index), 1000, null_p))
    check_against_plain(schema, batch, codec, mixed_sizes(schema), page_index, **SMALL)


@pytest.mark.parametrize("codec", [0, 6])
def test_slice_with_row0(codec):
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(3), 1200, 0.3))
    bloom = all_but_bool(schema, 1000, 0.01)
    check_against_plain(schema, batch, codec, bloom, 1, row0=136, n=900, **SMALL)
    check_against_plain(schema, batch, codec, bloom[::3], 0, row0=8, n=-1, page_rows=48, row_group_rows=100)


@pytest.mark.parametrize("codec", [0, 6])
def test_device_decoder_reads_files_with_filters(codec):
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(21), 5000, 0.4))
    bloom = mixed_sizes(schema)
    on, got = encode(schema, batch, codec, bloom, 1, page_rows=512, row_group_rows=2048, device_image=True)
    check_filters(on, batch, bloom, page_rows=512, row_group_rows=2048)
    assert got.equals(batch), got.first_difference(batch)
    back = arrow_to_batch(schema, pq.read_table(pa.BufferReader(on)))
    assert back.equals(batch), back.first_difference(batch)


@pytest.mark.parametrize("codec", [0, 6])
def test_no_bloom_columns_write_the_compressed_bytes(codec):
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(8), 700, 0.2))
    want = encode(schema, batch, codec, "compressed", 1, **SMALL)
    assert encode(schema, batch, codec, None, 1, **SMALL) == want
    assert encode(schema, batch, codec, [], 1, **SMALL) == want
    assert encode(schema, batch, codec, None, 1, raw_bloom=N.PgParquetBloomOptions(0, None), **SMALL) == want


def test_refusals():
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(2), 50))
    nc = schema.n_cols

    def status(bloom=None, codec=0, level=1, raw=None):
        try:
            encode(schema, batch, codec, bloom, raw_bloom=raw, level=level)
            return 0
        except N.PaimonGpuError as e:
            return e.status
    assert status([(3, 1000, 0.01)]) == 0
    invalid = [[(-1, 0, 0.01)], [(nc, 0, 0.01)], [(3, 0, 0.01), (3, 10, 0.1)], [(3, -1, 0.01)], [(3, 0, 0.0)],
               [(3, 0, 1.0)], [(3, 10, float("nan"))], [(3, 10, -0.5)]]
    for bloom in invalid:
        assert status(bloom) == 1, bloom
    assert status(raw=N.PgParquetBloomOptions(-1, None)) == 1
    assert status(raw=N.PgParquetBloomOptions(2, None)) == 1
    assert status([(BOOL_COL, 0, 0.01)]) == 2
    assert status([(3, 0, 0.01), (BOOL_COL, 100, 0.01)]) == 2
    # codecs and levels as pg_parquet_encode_compressed refuses them
    assert status([(3, 0, 0.01)], codec=1) == 2
    assert status([(3, 0, 0.01)], codec=99) == 1
    assert status([(3, 0, 0.01)], codec=6, level=3) == 2


def _bool_files(tmp_path, schema):
    """Two overlapping sorted input files of all_types_schema rows (BOOLEAN value field included)."""
    metas = []
    for f in range(2):
        rows = []
        for r in random_rows(random.Random(40 + f), 3000, 0.3):
            k = 2 * r[0] + f
            rows.append((k, r[1] + f, 0, k) + tuple(r[4:]))
        batch = KeyValueBatch.from_rows(schema, rows)
        path = str(tmp_path / f"in-{f}.parquet")
        write_kv_parquet(batch, path)
        metas.append(DataFileMeta(path, 0, batch.n_rows, rows[0][0], rows[-1][0], level=0))
    return metas


def test_compact_rewriter_enable_bloom_filter(tmp_path):
    """ParquetFormatReadWriteTest.testEnableBloomFilter restated: with 'parquet.bloom.filter.enabled' every column
    chunk of every written file has a filter, BOOLEAN ones excepted; without, none has; ORC levels are unaffected."""
    schema = all_types_schema()
    metas = _bool_files(tmp_path, schema)
    sections = IntervalPartition(metas).partition()
    factory = DeduplicateMergeFunction.factory()
    base = {"file.format": "parquet", "file.format.per.level": "5:orc", "file.compression": "zstd"}
    out = {}
    for flag in ("true", "false", None):
        options = dict(base) if flag is None else dict(base, **{"parquet.bloom.filter.enabled": flag})
        for level in (1, 5):
            d = tmp_path / f"{flag}-{level}"
            os.makedirs(str(d))
            res = MergeTreeCompactRewriter(schema, factory, str(d), target_file_rows=2000, page_rows=512,
                                           options=options).rewrite_compaction(level, False, sections)
            out[flag, level] = [open(m.file_name, "rb").read() for m in res.after]
    assert len(out["true", 1]) > 1
    bloom = all_but_bool(schema)
    for data in out["true", 1]:
        filters = R.file_filters(data)
        for row in filters:
            assert [c for c, f in enumerate(row) if f is None] == [BOOL_COL]
        batch = arrow_to_batch(schema, pq.read_table(pa.BufferReader(data)))
        check_filters(data, batch, bloom, page_rows=512)
    assert out["false", 1] == out[None, 1]
    for data in out["false", 1]:
        assert all(f is None for row in R.file_filters(data) for f in row)
    assert out["true", 5] == out["false", 5] == out[None, 5]
    assert all(d[:3] == b"ORC" for d in out["true", 5])
