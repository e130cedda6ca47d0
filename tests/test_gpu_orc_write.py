"""Compaction output encode as ORC on the device (pg_orc_encode): every file is read back by pyarrow.orc and by the
device's own ORC decoder (pg_orc_read_section) and must equal the source batch bit for bit; the footers' stripe and file
statistics match orc_stats_reference's model, and so do pg_parquet_file_column_stats / pg_parquet_file_meta; the
refusals; MergeTreeCompactRewriter with 'file.format' = orc and with 'file.format.per.level' mixing formats."""
import ctypes as C
import os
import random

import numpy as np
import pyarrow as pa
import pyarrow.orc as orc
import pytest

import orc_stats_reference as ref
from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import Column, KeyValueBatch, unpack_validity
from paimon_b200.compact_rewriter import KeyValueDataFileWriter, MergeTreeCompactRewriter, file_column_names
from paimon_b200.format import FileFormat, FormatReaderContext, LocalFileIO
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.merge_tree_readers import DataFileMeta, IntervalPartition, MergeFileSplitRead, concat_batches
from paimon_b200.sort_merge_reader import SortedRunReader, SortMergeReader, _SchemaHandle
from paimon_b200.types import DataField, KeyValueSchema, RowType, is_varlen, orc_column_type

from parquet_util import arrow_to_column, write_kv_parquet

pytestmark = pytest.mark.gpu


def all_types_schema():
    vt = RowType((DataField("pk", "INT", False), DataField("t", "TINYINT", True), DataField("s", "SMALLINT", True),
                  DataField("i", "INT", True), DataField("l", "BIGINT", True), DataField("f", "FLOAT", True),
                  DataField("d", "DOUBLE", True), DataField("str", "STRING", True), DataField("vc", "VARCHAR(6)", True),
                  DataField("bin", "BINARY(4)", True), DataField("b", "BOOLEAN", True), DataField("dt", "DATE", True),
                  DataField("dec", "DECIMAL(15,4)", True), DataField("nn", "BIGINT", False)))
    return KeyValueSchema.of(vt, ["pk"])


def random_rows(rng, n, null_p):
    rows = []
    for k in range(n):
        def opt(v):
            return None if rng.random() < null_p else v
        f = rng.choice([np.float32(rng.uniform(-1e3, 1e3)).item(), 0.0, -0.0])
        rows.append((k, k * 3 + 1, rng.choice([0, 1, 2, 3]), k, opt(rng.randrange(-128, 128)),
                     opt(rng.randrange(-32768, 32768)), opt(rng.choice([7, rng.randrange(-2 ** 31, 2 ** 31)])),
                     opt(rng.choice([k * 1000, rng.randrange(-2 ** 63, 2 ** 63)])), opt(f),
                     opt(rng.uniform(-1e9, 1e9)), opt("".join(rng.choice("abcé€") for _ in range(rng.randrange(0, 30)))),
                     opt("".join(rng.choice("xyé") for _ in range(rng.randrange(0, 7)))),
                     opt(bytes(rng.randrange(256) for _ in range(rng.randrange(0, 9)))), opt(rng.random() < 0.5),
                     opt(rng.randrange(-10000, 30000)), opt(rng.randrange(-10 ** 14, 10 ** 14)),
                     rng.randrange(-10 ** 12, 10 ** 12)))
    return rows


def orc_table_to_batch(schema, table):
    cols = []
    for f, name in zip(schema.file_fields(), table.column_names):
        arr = table.column(name).combine_chunks()
        if pa.types.is_date32(arr.type):
            arr = arr.cast(pa.int32())
        if pa.types.is_decimal(arr.type):
            vals = [None if v is None else int(v.scaleb(arr.type.scale)) for v in arr.to_pylist()]
            cols.append(Column.from_pylist(f.physical, vals))
        else:
            cols.append(arrow_to_column(f.physical, arr))
    return KeyValueBatch(schema, cols)


def encode(schema, batch, path, row0=0, n_rows=-1, **writer_args):
    """host batch -> device run -> pg_orc_encode of rows [row0, row0 + n_rows) -> file"""
    N.init(0)
    sh = _SchemaHandle(schema, 0)
    rd = SortedRunReader(schema, batch)
    try:
        h = rd._open(sh.handle)
        return KeyValueDataFileWriter(schema, path, level=0, file_format="orc", **writer_args).write(h, row0, n_rows)
    finally:
        rd.close()
        sh.close()


def read_device(schema, path):
    rd = FileFormat.from_identifier("orc").create_reader_factory(schema).create_reader(FormatReaderContext(LocalFileIO(), path))
    try:
        return rd.read_batch()
    finally:
        rd.close()


def slice_batch(schema, batch, r0, r1):
    return KeyValueBatch.from_rows(schema, batch.to_rows()[r0:r1])


def model_columns(schema, batch):
    out = []
    for f, col in zip(schema.file_fields(), batch.columns):
        kind, _, scale, _ = orc_column_type(f.type)
        n = len(col)
        valid = np.ones(n, bool) if col.valid is None else unpack_validity(col.valid, n)
        vals = [b"" if v is None else (v.encode() if isinstance(v, str) else v) for v in col.to_pylist()] \
            if is_varlen(col.type) else np.asarray(col.data[:n])
        out.append((kind, vals, valid, scale))
    return out


def check_file(schema, batch, path, written, stripe_rows):
    n = batch.n_rows
    table = orc.ORCFile(path).read()
    assert table.column_names == file_column_names(schema)
    got = orc_table_to_batch(schema, table)
    assert got.equals(batch), got.first_difference(batch)
    if n:
        dev = read_device(schema, path)
        assert dev.equals(batch), dev.first_difference(batch)
    assert written.meta.row_count == n
    sr = ((stripe_rows or (1 << 20)) + 7) & ~7
    kinds = np.asarray(batch.columns[schema.n_key + 1].data[:n])
    assert written.meta.delete_row_count == int(np.isin(kinds, [1, 3]).sum())
    if n:
        seq = np.asarray(batch.columns[schema.n_key].data[:n])
        assert (written.meta.min_sequence_number, written.meta.max_sequence_number) == (int(seq.min()), int(seq.max()))
    # pg_parquet_file_column_stats of the value columns
    model = model_columns(schema, batch)
    for c, st in enumerate(written.value_stats):
        kind, vals, valid, _ = model[schema.n_key + 2 + c]
        assert st.null_count == int((~valid).sum())
        fixed = not isinstance(vals, list)
        v = np.asarray(vals)[valid] if fixed else None
        if not fixed or not valid.any() or (v.dtype.kind == "f" and np.isnan(v).any()):
            assert st.min is None and st.max is None
        else:
            assert st.min == v.min() and st.max == v.max()
    # footer statistics (an uncompressed tail): stripes and file
    blob = open(path, "rb").read()
    ps = {f: v for f, _, v in ref.fields(blob[-1 - blob[-1]:-1])}
    if ps.get(2, 0) == 0:
        _, _, stripes, whole = ref.read_tail(blob)
        want_s, want_f = ref.expected(model, n, sr)
        assert len(stripes) == len(want_s)
        for g, (a_s, b_s) in enumerate(zip(stripes, want_s)):
            for c, (a, b) in enumerate(zip(a_s, b_s)):
                assert ref.same(a, b), (g, c, a, b)
        for c, (a, b) in enumerate(zip(whole, want_f)):
            assert ref.same(a, b), (c, a, b)


@pytest.mark.parametrize("n", [0, 1, 9, 1000, 4097])
@pytest.mark.parametrize("null_p", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("writer_args", [dict(), dict(stripe_rows=8), dict(stripe_rows=256, compression="zstd"),
                                         dict(stripe_rows=1000, compression="zstd", compression_block_size=2000)])
def test_every_type_round_trips(tmp_path, n, null_p, writer_args):
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(n * 7 + int(null_p * 10)), n, null_p))
    path = str(tmp_path / "out.orc")
    written = encode(schema, batch, path, **writer_args)
    check_file(schema, batch, path, written, writer_args.get("stripe_rows", 0))


@pytest.mark.parametrize("compression", ["none", "zstd"])
def test_slices_of_a_run_and_of_a_merge(tmp_path, compression):
    schema = datagen.schema_c3(n_i64=3, n_f64=2, n_str=3)
    run = datagen.make_runs(schema, 1, 30000, seed=4, null_prob=0.4, delete_prob=0.1)[0]
    n = run.n_rows
    for r0, cnt in [(0, -1), (16, 1000), (8, 0), (n - n % 8 - 8, -1)]:
        path = str(tmp_path / f"s{r0}.orc")
        written = encode(schema, run, path, r0, cnt, stripe_rows=4096, compression=compression)
        r1 = n if cnt < 0 else r0 + cnt
        check_file(schema, slice_batch(schema, run, r0, r1), path, written, 4096)
    # a merge handle holding a batch
    runs = datagen.make_runs(schema, 3, 20000, seed=5, null_prob=0.3)
    rd = SortMergeReader.create_sort_merge_reader([SortedRunReader(schema, b) for b in runs], None, None,
                                                  DeduplicateMergeFunction.factory().create())
    try:
        rd.execute()
        merged = rd.fetch()
        path = str(tmp_path / "merged.orc")
        written = KeyValueDataFileWriter(schema, path, 1, file_format="orc", stripe_rows=2048,
                                         compression=compression).write(rd._merge_h, 24, 5000)
    finally:
        rd.close()
    check_file(schema, slice_batch(schema, merged, 24, 5024), path, written, 2048)


def test_accessors_and_nan_statistics(tmp_path):
    vt = RowType((DataField("pk", "BIGINT", False), DataField("d", "DOUBLE", True), DataField("f", "FLOAT", True),
                  DataField("allnull", "BIGINT", True)))
    schema = KeyValueSchema.of(vt, ["pk"])
    rows = [(k, k, 0, k, float("nan") if k == 50 else -0.0 if k % 2 else float(k), 0.0, None) for k in range(100)]
    batch = KeyValueBatch.from_rows(schema, rows)
    path = str(tmp_path / "nan.orc")
    written = encode(schema, batch, path, stripe_rows=40)
    check_file(schema, batch, path, written, 40)
    _, _, stripes, whole = ref.read_tail(open(path, "rb").read())
    d, f, allnull = 5, 6, 7                                           # [root, _KEY_pk, seq, kind, pk, d, f, allnull]
    assert np.isnan(whole[d]["max"]) and whole[d]["min"] == -np.inf
    assert not np.isnan(stripes[0][d]["max"]) and np.isnan(stripes[1][d]["max"])   # only stripes holding a NaN
    assert whole[allnull] == {"values": 0, "has_null": True}
    assert np.signbit(whole[f]["min"]) and not np.signbit(whole[f]["max"])
    assert written.value_stats[1].min is None                                       # d holds a NaN
    assert written.value_stats[2].min == 0.0 and np.signbit(written.value_stats[2].min)
    assert written.n_pages > 0 and written.meta.file_size == os.path.getsize(path)


def _chunks(blob, block):
    """(original, length, offset) of every compression chunk between the magic and the PostScript: the streams, the
    stripe footers, the Metadata and the Footer, back to back"""
    end = len(blob) - 1 - blob[-1]
    pos, out = 3, []
    while pos < end:
        h = blob[pos] | blob[pos + 1] << 8 | blob[pos + 2] << 16
        length = h >> 1
        assert 0 < length <= block and pos + 3 + length <= end, (pos, length)
        out.append((h & 1, length, pos + 3))
        pos += 3 + length
    assert pos == end
    return out


def _zstd_blocks(frame):
    """the number of blocks of one zstd frame (RFC 8878), which has to fill `frame` exactly"""
    assert frame[:4] == b"\x28\xb5\x2f\xfd"
    fhd = frame[4]
    single = fhd >> 5 & 1
    pos = 5 + (1 - single) + (0, 1, 2, 4)[fhd & 3] + (single, 2, 4, 8)[fhd >> 6]
    n = 0
    while True:
        h = frame[pos] | frame[pos + 1] << 8 | frame[pos + 2] << 16
        pos += 3 + (1 if (h >> 1 & 3) == 1 else h >> 3)             # an RLE block holds one byte
        n += 1
        if h & 1:
            break
    assert pos + 4 * (fhd >> 2 & 1) == len(frame)
    return n


def test_zstd_chunks_stored_original_and_compressed(tmp_path):
    """ORC ZSTD chunks as the device gathers them.  Under a 4096-byte block, random bytes are stored as original
    chunks and a repeated string as compressed ones.  Under the default 256 KiB block, the 400 KB stream of the
    repeated string has a chunk whose frame holds two zstd blocks, and the random one an original chunk longer than a
    block.  Every chunk header is walked; the files read back through pyarrow.orc and the device decoder."""
    vt = RowType((DataField("pk", "INT", False), DataField("rnd", "BYTES", False), DataField("rep", "STRING", False)))
    schema = KeyValueSchema.of(vt, ["pk"])
    rng = random.Random(11)
    n = 8000
    batch = KeyValueBatch.from_rows(schema, [(k, k + 1, 0, k, rng.randbytes(50), "paimon-orc" * 5) for k in range(n)])
    for block in (4096, 0):
        path = str(tmp_path / f"block{block}.orc")
        written = encode(schema, batch, path, compression="zstd", compression_block_size=block)
        check_file(schema, batch, path, written, 0)
        chunks = _chunks(open(path, "rb").read(), block or 256 << 10)
        assert any(orig for orig, _, _ in chunks) and any(not orig for orig, _, _ in chunks), block
        if not block:
            blob = open(path, "rb").read()
            assert any(not orig and _zstd_blocks(blob[at:at + ln]) >= 2 for orig, ln, at in chunks)
            assert any(orig and ln > 128 << 10 for orig, ln, _ in chunks)


def test_refusals():
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(5), 100, 0.2))
    lib = N.init(0)
    names = file_column_names(schema)
    arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
    fields = schema.file_fields()
    base = [orc_column_type(f.type) for f in fields]

    def run(h, row0=0, n_rows=-1, compression=0, level=1, block=0, types=None):
        t = (N.PgOrcColumnType * len(base))(*[N.PgOrcColumnType(*x) for x in (types or base)])
        opts = N.PgOrcWriteOptions(0, compression, level, block, t)
        fh = C.c_uint64(0)
        st = lib.pg_orc_encode(h, arr, row0, n_rows, C.byref(opts), C.byref(fh))
        if st == 0:
            lib.pg_parquet_file_free(fh.value)
        return st

    def with_type(c, t):
        ts = list(base)
        ts[c] = t
        return ts

    sh = _SchemaHandle(schema, 0)
    rd = SortedRunReader(schema, batch)
    mask = [f.name in ("pk", "i") for f in schema.value_type.fields]
    merge = SortMergeReader([SortedRunReader(schema, batch)], DeduplicateMergeFunction.factory().create()
                            .with_read_fields(mask))
    try:
        h = rd._open(sh.handle)
        merge.execute()
        col = {f.name: i for i, f in enumerate(fields)}
        assert run(h) == 0 and run(h, compression=5) == 0 and run(h, compression=5, level=-5) == 0
        for kind in (1, 2, 3, 4, 6):                                       # ZLIB SNAPPY LZO LZ4 BROTLI
            assert run(h, compression=kind) == 2
        assert run(h, compression=7) == 1 and run(h, compression=-1) == 1
        assert run(h, compression=5, level=0) == 2 and run(h, compression=5, level=3) == 2
        assert run(h, block=1 << 23) == 1 and run(h, block=-1) == 1 and run(h, compression=5, block=(1 << 23) - 1) == 0
        assert run(h, types=with_type(col["l"], (9, 0, 0, 0))) == 2       # TIMESTAMP
        assert run(h, types=with_type(col["str"], (17, 0, 0, 5))) == 2    # CHAR
        assert run(h, types=with_type(col["l"], (10, 0, 0, 0))) == 2      # LIST
        assert run(h, types=with_type(col["l"], (3, 0, 0, 0))) == 1       # INT over a BIGINT column
        assert run(h, types=with_type(col["dec"], (14, 19, 2, 0))) == 1   # DECIMAL(19) does not fit int64
        assert run(h, types=with_type(col["str"], (8, 0, 0, 0))) == 1     # BINARY over a string column
        assert run(h, types=with_type(col["l"], (99, 0, 0, 0))) == 1
        assert run(h, types=with_type(col["vc"], (16, 0, 0, 2))) == 2     # a value longer than VARCHAR(2)
        assert run(h, types=with_type(col["vc"], (16, 0, 0, 6))) == 0
        assert run(h, row0=3) == 1 and run(h, row0=0, n_rows=101) == 1
        assert run(merge._merge_h) == 1                                    # projected batch
    finally:
        rd.close()
        merge.close()
        sh.close()


def _files(tmp_path, schema, ranges, nfiles, seed):
    rng = np.random.default_rng(seed)
    metas, file_runs = [], []
    for lo, hi in ranges:
        for f in range(nfiles):
            keys = np.sort(rng.choice(np.arange(lo, hi), size=int((hi - lo) * 0.4), replace=False)).astype(np.int64)
            file_runs.append(datagen.make_run(schema, len(file_runs), keys, seed=3, null_prob=0.3, delete_prob=0.15))
    for i, run in enumerate(file_runs):
        path = str(tmp_path / f"in-{i}.parquet")
        write_kv_parquet(run, path)
        k = run.columns[0].data
        metas.append(DataFileMeta(path, 0, run.n_rows, int(k[0]), int(k[-1]), level=0))
    return metas, file_runs


def _read_all(schema, factory, metas):
    rd = MergeFileSplitRead(schema, factory).create_merge_reader(metas, keep_delete=True)
    batches = []
    while True:
        b = rd.read_batch()
        if b is None:
            break
        batches.append(b)
    rd.close()
    return concat_batches(schema, batches)


@pytest.mark.parametrize("options", [{"file.format": "orc", "file.compression": "none"},
                                     {"file.format": "orc"},
                                     {"file.format": "parquet", "file.format.per.level": "5:orc,1:parquet",
                                      "orc.compress.size": "4096"}])
def test_compact_rewriter_writes_orc(tmp_path, options):
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    metas, file_runs = _files(tmp_path, schema, [(0, 4000), (6000, 9000)], 4, 7)
    factory = DeduplicateMergeFunction.factory()
    rewriter = MergeTreeCompactRewriter(schema, factory, str(tmp_path), target_file_rows=1000, options=options)
    result = rewriter.rewrite_compaction(5, False, IntervalPartition(metas).partition())
    assert result.after and all(m.file_name.endswith(".orc") for m in result.after)
    want = pyoracle.merge(schema, factory.create(), file_runs)
    got = _read_all(schema, factory, result.after)
    assert got.equals(want), got.first_difference(want)
    if "file.format.per.level" in options:
        os.makedirs(str(tmp_path / "l1"))
        again = MergeTreeCompactRewriter(schema, factory, str(tmp_path / "l1"), target_file_rows=1500, options=options)
        res1 = again.rewrite_compaction(1, False, IntervalPartition(metas).partition())
        assert all(m.file_name.endswith(".parquet") for m in res1.after)
        got1 = _read_all(schema, factory, res1.after)
        assert got1.equals(want), got1.first_difference(want)


def test_compact_rewriter_refuses_other_formats_before_device_work(tmp_path):
    schema = datagen.schema_c3(n_i64=1, n_f64=1, n_str=1)
    rewriter = MergeTreeCompactRewriter(schema, DeduplicateMergeFunction.factory(), str(tmp_path),
                                        options={"file.format": "orc", "file.format.per.level": "0:avro"})
    with pytest.raises(N.UnsupportedOnDevice):
        rewriter.rewrite_compaction(0, False, [])
