"""The Parquet page index of the files the device encoder writes (pg_parquet_write_options.page_index = 1), against
the independent model (tests/page_index_reference.py): pyarrow sees an OffsetIndex on every chunk and a ColumnIndex on
every chunk without a NaN, both structures equal the model's exactly, every page location points at a page header
that agrees with it, the file up to the index is the index-off file byte for byte, and both pyarrow and the device's
own decoder read the indexed file as they read the plain one.  Uncompressed and zstd.  Needs an H100."""
import ctypes as C
import random

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import page_index_reference as P
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import KeyValueBatch
from paimon_b200.compact_rewriter import MergeTreeCompactRewriter, file_column_names
from paimon_b200.format import FileFormat, FormatReaderContext, LocalFileIO, read_section
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.merge_tree_readers import DataFileMeta, IntervalPartition
from paimon_b200.sort_merge_reader import SortedRunReader, _SchemaHandle
from paimon_b200.types import DataField, KeyValueSchema, RowType

from parquet_util import arrow_to_batch, write_kv_parquet
from test_gpu_parquet_write import all_types_schema, random_rows

pytestmark = pytest.mark.gpu

CODECS = [None, 6]                                   # pg_parquet_encode, pg_parquet_encode_compressed ZSTD
SMALL = dict(page_rows=64, row_group_rows=256)


def encode(schema, batch, codec, page_index, row0=0, n=-1, page_rows=0, row_group_rows=0, device_image=False):
    """-> file bytes (and, with device_image, the bytes of pg_parquet_file_device_image decoded by the device)."""
    lib = N.init(0)
    sh = _SchemaHandle(schema, 0)
    rd = SortedRunReader(schema, batch)
    names = file_column_names(schema)
    arr = (C.c_char_p * len(names))(*[x.encode() for x in names])
    opts = N.PgParquetWriteOptions(row_group_rows, page_rows, page_index)
    fh = C.c_uint64(0)
    try:
        h = rd._open(sh.handle)
        if codec is None:
            N.check(lib.pg_parquet_encode(h, arr, row0, n, C.byref(opts), C.byref(fh)))
        else:
            N.check(lib.pg_parquet_encode_compressed(h, arr, row0, n, C.byref(opts), codec, 1, C.byref(fh)))
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


def check_page_index(file_bytes, batch, row0=0, n=-1, **writer_args):
    """Holds the page index of `file_bytes` to the model; returns the offset of the first index byte."""
    want = P.page_index(batch, row0, n, **writer_args)
    md = pq.ParquetFile(pa.BufferReader(file_bytes)).metadata
    refs = P.footer_chunks(file_bytes)
    assert md.num_row_groups == len(want) == len(refs)
    first = len(file_bytes)
    for g, (wrow, rrow) in enumerate(zip(want, refs)):
        for c, (w, r) in enumerate(zip(wrow, rrow)):
            where = f"row group {g} column {c}"
            cc = md.row_group(g).column(c)
            assert cc.has_offset_index, where
            assert cc.has_column_index == (w.column_index is not None), where
            assert (r.column_index is None) == (w.column_index is None), where
            if r.column_index is not None:
                off, ln = r.column_index
                assert P.parse_column_index(file_bytes[off:off + ln]) == w.column_index, where
                first = min(first, off)
            off, ln = r.offset_index
            first = min(first, off)
            locs = P.parse_offset_index(file_bytes[off:off + ln])
            assert [x[2] for x in locs] == [p for p, _ in w.pages], where
            # the locations cover exactly the chunk's pages, each at a header that agrees with it
            pos = r.data_page_offset
            for (loc_off, size, _), (_, rows) in zip(locs, w.pages):
                assert loc_off == pos, where
                hb, stored, num_values = P.page_header(file_bytes, loc_off)
                assert (hb + stored, num_values) == (size, rows), where
                pos += size
            assert pos == r.data_page_offset + r.total_compressed_size, where
            assert sum(rows for _, rows in w.pages) == r.num_values, where
    # ColumnIndexes first, then OffsetIndexes, then the footer
    footer = len(file_bytes) - 8 - int.from_bytes(file_bytes[-8:-4], "little")
    spans = sorted([x for row in refs for r in row for x in (r.column_index, r.offset_index) if x is not None])
    assert spans[0][0] == first and all(a[0] + a[1] == b[0] for a, b in zip(spans, spans[1:]))
    assert spans[-1][0] + spans[-1][1] == footer
    ci = [r.column_index[0] for row in refs for r in row if r.column_index is not None]
    oi = [r.offset_index[0] for row in refs for r in row]
    assert ci == sorted(ci) and oi == sorted(oi) and (not ci or max(ci) < min(oi))
    return first


def check_against_index_off(schema, batch, codec, row0=0, n=-1, **writer_args):
    on = encode(schema, batch, codec, 1, row0, n, **writer_args)
    off = encode(schema, batch, codec, 0, row0, n, **writer_args)
    first = check_page_index(on, batch, row0, n, **writer_args)
    assert on[:first] == off[:first]
    assert all(r.offset_index is None and r.column_index is None for row in P.footer_chunks(off) for r in row)
    # (repr: NaN equals NaN, -0.0 differs from +0.0)
    assert repr(pq.read_table(pa.BufferReader(on)).to_pydict()) == repr(pq.read_table(pa.BufferReader(off)).to_pydict())
    return on


def _string_schema():
    vt = RowType((DataField("pk", "INT", False), DataField("s", "STRING", True), DataField("b", "BINARY", True)))
    return KeyValueSchema.of(vt, ["pk"])


@pytest.mark.parametrize("codec", CODECS)
@pytest.mark.parametrize("null_p", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("n, writer_args", [(1000, SMALL), (4097, {})])
def test_all_types(codec, null_p, n, writer_args):
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(n + int(10 * null_p)), n, null_p))
    check_against_index_off(schema, batch, codec, **writer_args)


@pytest.mark.parametrize("codec", CODECS)
def test_slice_with_row0(codec):
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(3), 1200, 0.3))
    check_against_index_off(schema, batch, codec, row0=136, n=900, **SMALL)
    check_against_index_off(schema, batch, codec, row0=8, n=-1, page_rows=48, row_group_rows=100)


def _long_values(rng, n):
    """STRING values around 64 bytes with 2-, 3- and 4-byte characters across byte 64, prefixes of each other, and
    BINARY values of 0xFF runs that cannot be incremented."""
    chars = ["a", "z", "\u00e9", "\u20ac", "\U0001f600", "\U0010ffff", "\x7f"]
    rows = []
    for k in range(n):
        lead = rng.randrange(58, 66)
        s = "m" * lead + "".join(rng.choice(chars) for _ in range(rng.randrange(0, 6)))
        if rng.random() < 0.1:
            s = s[:rng.randrange(0, len(s) + 1)]
        if rng.random() < 0.01:
            s = "\U0010ffff" * rng.randrange(16, 20)
        b = bytes([0xFF] * rng.randrange(60, 66) + [rng.randrange(256) for _ in range(rng.randrange(0, 100))])
        if rng.random() < 0.98:
            b = bytes(rng.randrange(256) for _ in range(rng.randrange(0, 100)))
        rows.append((k, k, 0, k, None if rng.random() < 0.2 else s, None if rng.random() < 0.2 else b))
    return rows


@pytest.mark.parametrize("codec", CODECS)
def test_long_strings_truncated_at_64_bytes(codec):
    schema = _string_schema()
    batch = KeyValueBatch.from_rows(schema, _long_values(random.Random(11), 2000))
    check_against_index_off(schema, batch, codec, **SMALL)
    idx = P.page_index(batch, **SMALL)
    for c in (4, 5):                                       # each column needed a max written whole, and truncated one
        maxes = [v for row in idx for v in row[c].column_index.max_values]
        assert any(len(v) > P.TRUNCATE + 1 for v in maxes) and any(0 < len(v) <= P.TRUNCATE for v in maxes)


def _float_schema():
    vt = RowType((DataField("pk", "INT", False), DataField("f", "FLOAT", True), DataField("d", "DOUBLE", True)))
    return KeyValueSchema.of(vt, ["pk"])


@pytest.mark.parametrize("codec", CODECS)
def test_signed_zero_and_nan_pages(codec):
    schema = _float_schema()
    rows = []
    for k in range(1024):
        page = k // 64
        if page % 4 == 0:
            f = d = -0.0 if k % 2 else 0.0                 # zeros only: min -0.0, max +0.0
        elif page % 4 == 1:
            f = d = float(k)
        elif page % 4 == 2:
            f, d = (-0.0, 0.0) if k % 3 else (None, None)
        else:
            f, d = float(-k), float(-k)
        rows.append((k, k, 0, k, f, d))
    rows[5 * 64 + 7] = rows[5 * 64 + 7][:5] + (float("nan"),)      # a NaN in the DOUBLE of row group 1 only
    batch = KeyValueBatch.from_rows(schema, rows)
    on = check_against_index_off(schema, batch, codec, **SMALL)
    md = pq.ParquetFile(pa.BufferReader(on)).metadata
    assert not md.row_group(1).column(5).has_column_index and md.row_group(0).column(5).has_column_index
    assert md.row_group(1).column(4).has_column_index and md.row_group(1).column(5).has_offset_index


@pytest.mark.parametrize("codec", CODECS)
def test_sorted_keys_are_ascending(codec):
    for schema in (datagen.schema_c3(n_i64=2, n_f64=1, n_str=2), _c4_schema()):
        run = datagen.make_runs(schema, 1, 20000, seed=9, null_prob=0.3, delete_prob=0.1)[0]
        check_against_index_off(schema, run, codec, page_rows=1000, row_group_rows=8000)
        on = encode(schema, run, codec, 1, page_rows=1000, row_group_rows=8000)
        for row in P.footer_chunks(on):
            off, ln = row[0].column_index
            assert P.parse_column_index(on[off:off + ln]).boundary_order == P.ASCENDING


def _c4_schema():
    """bench.py's C4 row: a VARCHAR(16) key, BIGINT / DOUBLE / INT / VARCHAR(64) values."""
    fields = [DataField("pk", "VARCHAR(16)", False)]
    fields += [DataField(f"i{i}", "BIGINT", True) for i in range(4)]
    fields += [DataField(f"d{i}", "DOUBLE", True) for i in range(2)]
    fields += [DataField(f"n{i}", "INT", True) for i in range(2)]
    fields += [DataField(f"s{i}", "VARCHAR(64)", True) for i in range(3)]
    return KeyValueSchema.of(RowType(tuple(fields)), ["pk"])


@pytest.mark.parametrize("codec", CODECS)
def test_device_decoder_reads_indexed_files(tmp_path, codec):
    schema = datagen.schema_c3(n_i64=3, n_f64=2, n_str=3)
    run = datagen.make_runs(schema, 1, 30000, seed=4, null_prob=0.4, delete_prob=0.1)[0]
    on, got_image = encode(schema, run, codec, 1, page_rows=4096, row_group_rows=16384, device_image=True)
    check_page_index(on, run, page_rows=4096, row_group_rows=16384)
    assert got_image.equals(run), got_image.first_difference(run)
    path = str(tmp_path / "indexed.parquet")
    with open(path, "wb") as f:
        f.write(on)
    rd = FileFormat.from_identifier("parquet").create_reader_factory(schema).create_reader(
        FormatReaderContext(LocalFileIO(), path))
    try:
        got = rd.read_batch()
    finally:
        rd.close()
    assert got.equals(run), got.first_difference(run)


def test_page_index_values_other_than_0_and_1_are_refused():
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(2), 50))
    for v in (-1, 2, 7):
        with pytest.raises(N.PaimonGpuError) as e:
            encode(schema, batch, None, v)
        assert e.value.status == 1 and not isinstance(e.value, N.UnsupportedOnDevice)


def test_compact_rewriter_indexes_parquet_levels_only(tmp_path):
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    rng = np.random.default_rng(7)
    metas = []
    for f in range(3):
        keys = np.sort(rng.choice(np.arange(0, 5000), size=2000, replace=False)).astype(np.int64)
        r = datagen.make_run(schema, f, keys, seed=3, null_prob=0.3, delete_prob=0.15)
        path = str(tmp_path / f"in-{f}.parquet")
        write_kv_parquet(r, path)
        metas.append(DataFileMeta(path, 0, r.n_rows, int(keys[0]), int(keys[-1]), level=0))
    factory = DeduplicateMergeFunction.factory()
    opts = {"file.format.per.level": "3:orc", "file.compression": "zstd"}
    outputs = {}
    for level, page_index in ((2, True), (3, True), (4, False)):
        out = tmp_path / f"l{level}-{page_index}"
        out.mkdir()
        rewriter = MergeTreeCompactRewriter(schema, factory, str(out), target_file_rows=1500, page_rows=256,
                                            options=opts, **({"page_index": True} if page_index else {}))
        outputs[level] = rewriter.rewrite_compaction(level, False, IntervalPartition(metas).partition())
    for m in outputs[2].after:
        data = open(m.file_name, "rb").read()
        batch = arrow_to_batch(schema, pq.read_table(m.file_name))
        check_page_index(data, batch, page_rows=256)
    # ORC level: the flag is ignored, the files are what the rewriter writes without it
    plain = tmp_path / "l3-plain"
    plain.mkdir()
    orc_plain = MergeTreeCompactRewriter(schema, factory, str(plain), target_file_rows=1500, page_rows=256,
                                         options=opts).rewrite_compaction(3, False, IntervalPartition(metas).partition())
    assert [open(m.file_name, "rb").read() for m in outputs[3].after] == \
        [open(m.file_name, "rb").read() for m in orc_plain.after]
    assert all(m.file_name.endswith(".orc") for m in outputs[3].after)
    # flag off (the default): no page index anywhere, pages run up to the footer
    for m in outputs[4].after:
        data = open(m.file_name, "rb").read()
        md = pq.ParquetFile(m.file_name).metadata
        assert not any(md.row_group(g).column(c).has_offset_index or md.row_group(g).column(c).has_column_index
                       for g in range(md.num_row_groups) for c in range(md.num_columns))
        end = len(data) - 8 - int.from_bytes(data[-8:-4], "little")
        i = 4
        while i < end:
            hb, stored, _ = P.page_header(data, i)
            i += hb + stored
        assert i == end
