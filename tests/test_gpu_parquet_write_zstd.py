"""zstd-compressed compaction output on the device (pg_parquet_encode_compressed, codec 6): the files read back with
pyarrow and with the device decoder, their footers carry ZSTD and both size totals, every frame decompresses on the
host to the body the uncompressed encode writes for that page and equals the frame the host build of the encoder
writes for that body, the bytes are deterministic, codec 0 is the
uncompressed encode, the refusals, the rewriter's per-level codec choice, and the ratio against libzstd level 1."""
import ctypes as C
import random

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import KeyValueBatch
from paimon_b200.compact_rewriter import MergeTreeCompactRewriter, compression_for_level, file_column_names
from paimon_b200.format import FileFormat, FormatReaderContext, LocalFileIO, read_section
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.merge_tree_readers import DataFileMeta, IntervalPartition, concat_batches
from paimon_b200.sort_merge_reader import SortedRunReader, _SchemaHandle
from paimon_b200.types import DataField, KeyValueSchema, RowType

from parquet_util import arrow_to_batch, write_kv_parquet
from test_gpu_parquet_write import all_types_schema, random_rows
from test_zstd_encode_cpu import compress, zse  # noqa: F401  (zse: the host build of the encoder, a fixture)

pytestmark = pytest.mark.gpu

ZSTD = pa.Codec("zstd", compression_level=1)


def encode(schema, batch, codec, level=1, page_rows=0, row_group_rows=0, keep_image=False):
    """host batch -> device run -> pg_parquet_encode(_compressed) -> (file bytes, pg_file_meta[, device image bytes])"""
    lib = N.init(0)
    sh = _SchemaHandle(schema, 0)
    rd = SortedRunReader(schema, batch)
    names = file_column_names(schema)
    arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
    opts = N.PgParquetWriteOptions(row_group_rows, page_rows)
    fh = C.c_uint64(0)
    try:
        h = rd._open(sh.handle)
        if codec is None:
            N.check(lib.pg_parquet_encode(h, arr, 0, -1, C.byref(opts), C.byref(fh)))
        else:
            N.check(lib.pg_parquet_encode_compressed(h, arr, 0, -1, C.byref(opts), codec, level, C.byref(fh)))
        try:
            meta = N.PgFileMeta()
            N.check(lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
            buf = np.zeros(max(meta.file_bytes, 1), np.uint8)
            N.check(lib.pg_parquet_file_fetch(fh.value, buf.ctypes.data, meta.file_bytes))
            out = bytes(buf[: meta.file_bytes])
            if keep_image:
                return out, meta, fh.value
            return out, meta
        finally:
            if not keep_image:
                lib.pg_parquet_file_free(fh.value)
    finally:
        rd.close()
        sh.close()


def _varint(b, i):
    v = s = 0
    while True:
        x = b[i]
        i += 1
        v |= (x & 0x7F) << s
        s += 7
        if x < 0x80:
            return v, i


def _page_header(b, i):
    """(type, uncompressed size, compressed size, end of header) of a PageHeader as this encoder writes it."""
    fields, last, depth = {}, [0], 0
    while True:
        h = b[i]
        i += 1
        if h == 0:
            last.pop()
            depth -= 1
            if depth < 0:
                return fields[1], fields[2], fields[3], i
            continue
        d, t = h >> 4, h & 15
        fid = last[-1] + d
        last[-1] = fid
        if t == 5:
            v, i = _varint(b, i)
            if depth == 0:
                fields[fid] = (v >> 1) ^ -(v & 1)
        elif t == 12:
            last.append(0)
            depth += 1
        else:
            raise AssertionError(f"unexpected Thrift type {t}")


def pages_of(file_bytes):
    """[(uncompressed size, stored bytes)] of every page, in file order."""
    flen = int.from_bytes(file_bytes[-8:-4], "little")
    end = len(file_bytes) - 8 - flen
    i, out = 4, []
    while i < end:
        _, unc, comp, i = _page_header(file_bytes, i)
        out.append((unc, file_bytes[i:i + comp]))
        i += comp
    assert i == end
    return out


def check_against_uncompressed(schema, batch, path, zse, **writer_args):
    """The zstd encode against the uncompressed one of the same batch; returns the zstd file's metadata.  `zse` is
    the host build of the frame encoder (test_zstd_encode_cpu): every device frame must equal its frame."""
    raw, raw_meta = encode(schema, batch, None, **writer_args)
    z, z_meta = encode(schema, batch, 6, **writer_args)
    z2, _ = encode(schema, batch, 6, **writer_args)
    assert z == z2                                                   # deterministic
    assert encode(schema, batch, 0, **writer_args)[0] == raw         # codec 0 = the uncompressed encode
    with open(path, "wb") as f:
        f.write(z)
    got = arrow_to_batch(schema, pq.read_table(path))
    assert got.equals(batch), got.first_difference(batch)
    # same bodies: every frame decompresses to the body the uncompressed encode wrote for that page
    rp, zp = pages_of(raw), pages_of(z)
    assert len(rp) == len(zp) == z_meta.n_pages
    for (ru, rbody), (zu, frame) in zip(rp, zp):
        assert ru == zu == len(rbody)
        assert ZSTD.decompress(frame, decompressed_size=zu, asbytes=True) == rbody
        assert compress(zse, rbody) == frame                        # the host build writes the same bytes
        assert len(frame) <= len(rbody) + 6 + 8 + 3 * (len(rbody) // (128 << 10) + 1)
    # metadata: codec, both totals, statistics identical to the uncompressed file's
    zm, rm = pq.ParquetFile(path).metadata, pq.ParquetFile(pa.BufferReader(raw)).metadata
    assert (z_meta.n_rows, z_meta.n_pages, z_meta.min_sequence_number, z_meta.max_sequence_number,
            z_meta.delete_row_count) == (raw_meta.n_rows, raw_meta.n_pages, raw_meta.min_sequence_number,
                                         raw_meta.max_sequence_number, raw_meta.delete_row_count)
    assert z_meta.file_bytes == len(z) and (z_meta.launches > raw_meta.launches or not rp)
    saved = 0
    for g in range(zm.num_row_groups):
        assert zm.row_group(g).total_byte_size == sum(zm.row_group(g).column(c).total_uncompressed_size
                                                      for c in range(zm.num_columns))
        for c in range(zm.num_columns):
            zc, rc = zm.row_group(g).column(c), rm.row_group(g).column(c)
            assert zc.compression == "ZSTD" and rc.compression == "UNCOMPRESSED"
            assert rc.total_uncompressed_size == rc.total_compressed_size
            saved += zc.total_uncompressed_size - zc.total_compressed_size
            assert zc.statistics == rc.statistics
    assert saved == sum(u - len(f) for u, f in zp)
    # the compressed totals are exactly the bytes of the column chunks
    starts = sorted((zm.row_group(g).column(c).data_page_offset, zm.row_group(g).column(c).total_compressed_size)
                    for g in range(zm.num_row_groups) for c in range(zm.num_columns))
    for (a, n), (b, _) in zip(starts, starts[1:]):
        assert a + n == b
    return z


@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 255, 1000, 4097])
@pytest.mark.parametrize("writer_args", [dict(), dict(page_rows=64, row_group_rows=256)])
def test_pyarrow_reads_zstd_pages_the_device_writes(tmp_path, zse, n, writer_args):
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(n + 17), n))
    check_against_uncompressed(schema, batch, str(tmp_path / "z.parquet"), zse, **writer_args)


def _bulk_schema():
    vt = RowType((DataField("pk", "BIGINT", False), DataField("v", "BIGINT", True), DataField("d", "DOUBLE", True),
                  DataField("s", "STRING", True), DataField("nul", "BIGINT", True), DataField("b", "BOOLEAN", True)))
    return KeyValueSchema.of(vt, ["pk"])


def _bulk_table(schema, n, seed):
    rng = np.random.default_rng(seed)
    names = file_column_names(schema)
    words = np.array([b"alpha", b"beta", b"gamma", b"delta", b"paimon", b"merge-tree"])
    pk = np.arange(n, dtype=np.int64)
    s = [b"%s-%d" % (words[i % 6], x) for i, x in enumerate(rng.integers(0, 1 << 20, n))]
    cols = [pa.array(pk), pa.array(pk + 1000), pa.array(np.zeros(n, np.int8)), pa.array(pk),
            pa.array(rng.integers(0, 1000, n) * 1_000_003, mask=rng.random(n) < 0.1),
            pa.array(rng.integers(0, 1 << 16, n) / 64.0), pa.array(s, pa.string()),
            pa.nulls(n, pa.int64()), pa.array(rng.random(n) < 0.3)]
    fields = [pa.field(nm, c.type, nullable=i >= schema.n_key + 2) for i, (nm, c) in enumerate(zip(names, cols))]
    return pa.Table.from_arrays(cols, schema=pa.schema(fields))


def test_large_pages_many_blocks_per_frame(tmp_path, zse):
    """8-byte pages over 128 KiB, multi-MiB string pages (many blocks per frame), all-NULL and BOOLEAN pages."""
    schema = _bulk_schema()
    batch = arrow_to_batch(schema, _bulk_table(schema, 300_000, 1))
    z = check_against_uncompressed(schema, batch, str(tmp_path / "big.parquet"), zse, page_rows=150_000)
    sizes = [u for u, _ in pages_of(z)]
    assert max(sizes) > 2 << 20 and sum(1 for s in sizes if s > 128 << 10) >= 8


def test_device_decoder_reads_zstd_pages_the_device_writes(tmp_path):
    schema = datagen.schema_c3(n_i64=3, n_f64=2, n_str=3)
    run = datagen.make_runs(schema, 1, 50000, seed=4, null_prob=0.4, delete_prob=0.1)[0]
    z, meta, fh = encode(schema, run, 6, page_rows=4096, row_group_rows=16384, keep_image=True)
    lib = N.load()
    try:
        path = str(tmp_path / "rt.parquet")
        with open(path, "wb") as f:
            f.write(z)
        rd = FileFormat.from_identifier("parquet").create_reader_factory(schema).create_reader(
            FormatReaderContext(LocalFileIO(), path))
        try:
            got = rd.read_batch()
        finally:
            rd.close()
        assert got.equals(run), got.first_difference(run)
        ptr, size = C.c_void_p(0), C.c_int64(0)
        N.check(lib.pg_parquet_file_device_image(fh, C.byref(ptr), C.byref(size)))
        assert size.value == len(z)
        readers, _ = read_section(schema, [((ptr.value, size.value), 0)], 1)
        try:
            got2 = readers[0].read_batch()
        finally:
            for r in readers:
                r.close()
        assert got2.equals(run), got2.first_difference(run)
    finally:
        lib.pg_parquet_file_free(fh)


def test_codecs_and_levels_that_are_refused():
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(1), 100))
    for codec in (1, 2, 3, 4, 5, 7):
        with pytest.raises(N.UnsupportedOnDevice):
            encode(schema, batch, codec)
    for codec in (-1, 8, 99):
        with pytest.raises(N.PaimonGpuError) as e:
            encode(schema, batch, codec)
        assert not isinstance(e.value, N.UnsupportedOnDevice)
    for level in (0, 2, 3, 9, 22):
        with pytest.raises(N.UnsupportedOnDevice, match="file.compression.zstd-level"):
            encode(schema, batch, 6, level=level)
    for level in (1, -1, -5):
        encode(schema, batch, 6, level=level)


def test_compression_for_level_follows_the_table_options():
    assert compression_for_level({}, 0) == ("zstd", 1)
    assert compression_for_level(None, 3) == ("zstd", 1)
    opts = {"file.compression.per.level": "5:zstd", "file.compression": "none"}
    assert compression_for_level(opts, 5) == ("zstd", 1) and compression_for_level(opts, 4) == ("none", 1)
    assert compression_for_level({"file.compression": "lz4", "parquet.compression": "ZSTD"}, 1)[0] == "zstd"
    assert compression_for_level({"file.compression.zstd-level": "-3"}, 1) == ("zstd", -3)
    assert compression_for_level({"file.compression.zstd-level": 3, "parquet.compression.codec.zstd.level": 1}, 1) \
        == ("zstd", 1)


def test_compact_rewriter_writes_zstd_at_the_configured_level(tmp_path):
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    rng = np.random.default_rng(7)
    metas, file_runs = [], []
    for f in range(4):
        keys = np.sort(rng.choice(np.arange(0, 6000), size=2400, replace=False)).astype(np.int64)
        file_runs.append(datagen.make_run(schema, f, keys, seed=3, null_prob=0.3, delete_prob=0.15))
        path = str(tmp_path / f"in-{f}.parquet")
        write_kv_parquet(file_runs[-1], path)
        k = file_runs[-1].columns[0].data
        metas.append(DataFileMeta(path, 0, file_runs[-1].n_rows, int(k[0]), int(k[-1]), level=0))
    factory = DeduplicateMergeFunction.factory()
    want = pyoracle.merge(schema, factory.create(), file_runs)
    opts = {"file.compression.per.level": "5:zstd", "file.compression": "none"}
    for level, codec in ((5, "ZSTD"), (2, "UNCOMPRESSED")):
        out = tmp_path / f"l{level}"
        out.mkdir()
        rewriter = MergeTreeCompactRewriter(schema, factory, str(out), target_file_rows=1500, page_rows=256,
                                            options=opts)
        result = rewriter.rewrite_compaction(level, False, IntervalPartition(metas).partition())
        got = concat_batches(schema, [arrow_to_batch(schema, pq.read_table(m.file_name)) for m in result.after])
        assert got.equals(want), got.first_difference(want)
        for m in result.after:
            md = pq.ParquetFile(m.file_name).metadata
            assert {md.row_group(g).column(c).compression for g in range(md.num_row_groups)
                    for c in range(md.num_columns)} == {codec}
            assert m.level == level


def _c5_schema():
    fields = [DataField("l_orderkey", "BIGINT", False), DataField("l_linenumber", "INT", False),
              DataField("l_partkey", "BIGINT", True), DataField("l_suppkey", "BIGINT", True),
              DataField("l_quantity", "BIGINT", True), DataField("l_extendedprice", "BIGINT", True),
              DataField("l_discount", "BIGINT", True), DataField("l_tax", "BIGINT", True),
              DataField("l_returnflag", "STRING", True), DataField("l_linestatus", "STRING", True),
              DataField("l_shipdate", "INT", True), DataField("l_commitdate", "INT", True),
              DataField("l_receiptdate", "INT", True), DataField("l_shipinstruct", "STRING", True),
              DataField("l_shipmode", "STRING", True), DataField("l_comment", "STRING", True)]
    return KeyValueSchema.of(RowType(tuple(fields)), ["l_orderkey", "l_linenumber"])


def test_ratio_against_libzstd_level1_on_the_c5_shape(tmp_path):
    """The lineitem-shaped columns (bench.py's C5 generators, DECIMAL / DATE in their INT64 / INT32 form): the
    device's frames total at most 1.15x what libzstd level 1 makes of the same page bodies."""
    import pyarrow.compute as pc
    schema = _c5_schema()
    n = 400_000
    rng = np.random.default_rng(5)
    idx = np.arange(n, dtype=np.int64)
    ok, ln = idx // 4, (idx % 4 + 1).astype(np.int32)
    flags = [np.array([b"A", b"N", b"R"]), np.array([b"F", b"O"])]
    instr = np.array([b"DELIVER IN PERSON", b"COLLECT COD", b"NONE", b"TAKE BACK RETURN"])
    modes = np.array([b"REG AIR", b"AIR", b"RAIL", b"SHIP", b"TRUCK", b"MAIL", b"FOB"])
    cols = [pa.array(ok), pa.array(ln), pa.array(np.arange(n, dtype=np.int64)), pa.array(np.zeros(n, np.int8)),
            pa.array(ok), pa.array(ln), pa.array(rng.integers(1, 20_000_000, n)), pa.array(rng.integers(1, 1_000_000, n))]
    cols += [pa.array(rng.integers(100, 5_000_000, n)) for _ in range(4)]
    cols += [pa.array(flags[0][rng.integers(0, 3, n)]).cast(pa.string()),
             pa.array(flags[1][rng.integers(0, 2, n)]).cast(pa.string())]
    ship = rng.integers(8000, 10600, n).astype(np.int32)
    cols += [pa.array(ship), pa.array(ship + 30), pa.array(ship + 45)]
    cols += [pa.array(instr[rng.integers(0, 4, n)]).cast(pa.string()),
             pa.array(modes[rng.integers(0, 7, n)]).cast(pa.string())]
    cols.append(pc.binary_join_element_wise(pa.array(rng.integers(0, 1 << 40, n)).cast(pa.string()),
                                            pa.array(rng.integers(0, 1 << 30, n)).cast(pa.string()), " carefully final "))
    names = file_column_names(schema)
    fields = [pa.field(nm, c.type, nullable=i >= schema.n_key + 2) for i, (nm, c) in enumerate(zip(names, cols))]
    batch = arrow_to_batch(schema, pa.Table.from_arrays(cols, schema=pa.schema(fields)))
    raw, _ = encode(schema, batch, None, page_rows=20_000)
    z, _ = encode(schema, batch, 6, page_rows=20_000)
    ours = sum(len(f) for _, f in pages_of(z))
    lib1 = sum(len(ZSTD.compress(b, asbytes=True)) for _, b in pages_of(raw))
    print(f"C5 page bodies: {sum(u for u, _ in pages_of(raw))} B -> device zstd {ours} B, libzstd-1 {lib1} B, "
          f"ratio {ours / lib1:.3f}")
    assert ours <= 1.15 * lib1
