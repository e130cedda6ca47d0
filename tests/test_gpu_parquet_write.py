"""Compaction output encode on the device: Parquet files written by pg_parquet_encode are read back with pyarrow
(format conformance oracle) and with the device decoder; DataFileMeta fields and column statistics are checked
against the batch; MergeTreeCompactRewriter end to end against the merge oracle.  The reference pins its writer
the same way — by round trips (paimon-format/.../parquet/ParquetReadWriteTest.java:203-258) and by
MergeTreeTestBase's write -> compact -> read model (paimon-core/.../mergetree/MergeTreeTestBase.java:205-240)."""
import ctypes as C
import random

import numpy as np
import pyarrow.parquet as pq
import pytest

from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import KeyValueBatch, unpack_validity
from paimon_b200.compact_rewriter import KeyValueDataFileWriter, MergeTreeCompactRewriter, file_column_names
from paimon_b200.format import FileFormat, FormatReaderContext, LocalFileIO
from paimon_b200.merge_function import DeduplicateMergeFunction, PartialUpdateMergeFunction
from paimon_b200.merge_tree_readers import DataFileMeta, IntervalPartition, concat_batches
from paimon_b200.sort_merge_reader import SortedRunReader, SortMergeReader, _SchemaHandle
from paimon_b200.types import DataField, KeyValueSchema, PhysicalType, RowType, is_varlen

from parquet_util import arrow_to_batch, write_kv_parquet

pytestmark = pytest.mark.gpu


def encode_host_batch(schema, batch, path, **writer_args):
    """host batch -> device run -> pg_parquet_encode -> file"""
    N.init(0)
    sh = _SchemaHandle(schema, 0)
    rd = SortedRunReader(schema, batch)
    try:
        h = rd._open(sh.handle)
        return KeyValueDataFileWriter(schema, path, level=0, **writer_args).write(h)
    finally:
        rd.close()
        sh.close()


def all_types_schema():
    vt = RowType((DataField("pk", "INT", False), DataField("t", "TINYINT", True), DataField("s", "SMALLINT", True),
                  DataField("i", "INT", True), DataField("f", "FLOAT", True), DataField("d", "DOUBLE", True),
                  DataField("str", "STRING", True), DataField("bin", "BINARY", True), DataField("b", "BOOLEAN", True),
                  DataField("nn", "BIGINT", False)))
    return KeyValueSchema.of(vt, ["pk"])


def random_rows(rng, n, null_p=0.25):
    rows = []
    for k in range(n):
        def opt(v):
            return None if rng.random() < null_p else v
        rows.append((k, k * 3 + 1, rng.choice([0, 1, 2, 3]), k, opt(rng.randrange(-128, 128)),
                     opt(rng.randrange(-32768, 32768)), opt(rng.randrange(-2 ** 31, 2 ** 31)),
                     opt(np.float32(rng.uniform(-1e3, 1e3)).item()), opt(rng.uniform(-1e9, 1e9)),
                     opt("".join(rng.choice("abcdefgh") for _ in range(rng.randrange(0, 40)))),
                     opt(bytes(rng.randrange(256) for _ in range(rng.randrange(0, 20)))), opt(rng.random() < 0.5),
                     rng.randrange(-10 ** 12, 10 ** 12)))
    return rows


@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 255, 1000, 4097])
@pytest.mark.parametrize("writer_args", [dict(), dict(page_rows=64, row_group_rows=256)])
def test_pyarrow_reads_what_the_device_writes(tmp_path, n, writer_args):
    schema = all_types_schema()
    rng = random.Random(n + 17)
    batch = KeyValueBatch.from_rows(schema, random_rows(rng, n))
    path = str(tmp_path / "out.parquet")
    written = encode_host_batch(schema, batch, path, **writer_args)
    table = pq.read_table(path)
    assert table.column_names == file_column_names(schema)
    got = arrow_to_batch(schema, table)
    assert got.equals(batch), got.first_difference(batch)
    meta = pq.ParquetFile(path).metadata
    assert meta.num_rows == n and written.meta.row_count == n
    if writer_args and n:
        assert meta.num_row_groups == -(-n // 256)
    # DataFileMeta fields (KeyValueDataFileWriter.result, KeyValueDataFileWriter.java:150-184)
    kinds = np.asarray(batch.columns[2].data[:n])
    assert written.meta.delete_row_count == int(np.isin(kinds, [1, 3]).sum())
    if n:
        assert (written.meta.min_key, written.meta.max_key) == (0, n - 1)
        seq = np.asarray(batch.columns[1].data[:n])
        assert (written.meta.min_sequence_number, written.meta.max_sequence_number) == (int(seq.min()), int(seq.max()))
    # per-column statistics: ours and the ones pyarrow parses from the footer
    for ci, col in enumerate(batch.columns[3:]):
        st = written.value_stats[ci]
        valid = np.ones(n, bool) if col.valid is None else unpack_validity(col.valid, n)
        assert st.null_count == int((~valid).sum())
        if not is_varlen(col.type) and valid.any():
            vals = np.asarray(col.data[:n])[valid]
            assert st.min == vals.min() and st.max == vals.max()
    if n:
        rg = meta.row_group(0)
        for c in range(rg.num_columns):
            cs = rg.column(c).statistics
            assert cs is not None and cs.null_count is not None


def test_device_decoder_reads_what_the_device_writes(tmp_path):
    schema = datagen.schema_c3(n_i64=3, n_f64=2, n_str=3)
    run = datagen.make_runs(schema, 1, 50000, seed=4, null_prob=0.4, delete_prob=0.1)[0]
    path = str(tmp_path / "rt.parquet")
    written = encode_host_batch(schema, run, path, page_rows=4096, row_group_rows=16384)
    n = run.n_rows
    pages_per_col = sum(-(-min(16384, n - g) // 4096) for g in range(0, n, 16384))
    assert written.n_pages == schema.n_cols * pages_per_col and written.meta.row_count == n
    fmt = FileFormat.from_identifier("parquet")
    rd = fmt.create_reader_factory(schema).create_reader(FormatReaderContext(LocalFileIO(), path))
    try:
        got = rd.read_batch()
    finally:
        rd.close()
    assert got.equals(run), got.first_difference(run)
    assert arrow_to_batch(schema, pq.read_table(path)).equals(run)


def test_encoder_refuses_bad_arguments():
    """Both entry points refuse, with PG_ERR_INVALID and the same message: a row range that does not start at a
    multiple of 8 (the definition levels are the batch's bitmap bytes) or leaves the batch, a batch merged under a
    read-type projection (it lacks columns a data file needs), and an unknown source handle."""
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(5), 100))
    lib = N.init(0)
    names = file_column_names(schema)
    arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
    opts = N.PgParquetWriteOptions(0, 0)

    def encode_both(source, row0, n_rows):
        out = []
        for codec in (None, 6):
            fh = C.c_uint64(0)
            if codec is None:
                st = lib.pg_parquet_encode(source, arr, row0, n_rows, C.byref(opts), C.byref(fh))
            else:
                st = lib.pg_parquet_encode_compressed(source, arr, row0, n_rows, C.byref(opts), codec, 1, C.byref(fh))
            out.append((st, lib.pg_last_error().decode() if st else ""))
            if st == 0:
                lib.pg_parquet_file_free(fh.value)
        return out

    mask = [f.name in ("pk", "i") for f in schema.value_type.fields]
    merge = SortMergeReader([SortedRunReader(schema, batch)], DeduplicateMergeFunction.factory().create()
                            .with_read_fields(mask))
    sh = _SchemaHandle(schema, 0)
    run, gone = SortedRunReader(schema, batch), SortedRunReader(schema, batch)
    try:
        merge.execute()
        assert merge.device_batch().n_rows > 0
        h = run._open(sh.handle)
        unknown = gone._open(sh.handle)
        gone.close()
        assert encode_both(h, 8, -1) == [(0, ""), (0, "")]
        bad_range = "parquet encode: row range outside the batch or not starting at a multiple of 8"
        cases = [(h, 3, -1, bad_range), (h, 3, 8, bad_range), (h, -8, 8, bad_range), (h, 0, 101, bad_range),
                 (h, 96, 8, bad_range),
                 (merge._merge_h, 0, -1, "parquet encode: the batch was produced under a read-type projection"),
                 (unknown, 0, -1, "unknown run / merge handle")]
        for source, row0, n_rows, message in cases:
            for st, msg in encode_both(source, row0, n_rows):
                assert st == 1 and msg.startswith(message), (row0, n_rows, st, msg)
    finally:
        run.close()
        merge.close()
        sh.close()


@pytest.mark.parametrize("drop_delete", [True, False])
def test_compact_rewriter_end_to_end(tmp_path, drop_delete):
    """files -> IntervalPartition sections -> device merge per section -> device Parquet encode -> DataFileMeta;
    reading the new files back gives the oracle's merge of the old ones, and the new files form one sorted run."""
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    rng = np.random.default_rng(7)
    metas, file_runs = [], []
    for lo, hi in [(0, 4000), (6000, 9000)]:
        for f in range(5):
            keys = np.sort(rng.choice(np.arange(lo, hi), size=int((hi - lo) * 0.4), replace=False)).astype(np.int64)
            file_runs.append(datagen.make_run(schema, len(file_runs), keys, seed=3, null_prob=0.3, delete_prob=0.15))
    for i, run in enumerate(file_runs):
        path = str(tmp_path / f"in-{i}.parquet")
        write_kv_parquet(run, path, use_dictionary=(i % 2 == 0))
        k = run.columns[0].data
        metas.append(DataFileMeta(path, 0, run.n_rows, int(k[0]), int(k[-1]), level=0))
    factory = DeduplicateMergeFunction.factory()
    rewriter = MergeTreeCompactRewriter(schema, factory, str(tmp_path), target_file_rows=1000, page_rows=256)
    sections = IntervalPartition(metas).partition()
    assert len(sections) == 2
    result = rewriter.rewrite_compaction(5, drop_delete, sections)
    assert sorted(m.file_name for m in result.before) == sorted(m.file_name for m in metas)
    want = pyoracle.merge(schema, factory.create().with_drop_delete(drop_delete), file_runs)
    got = concat_batches(schema, [arrow_to_batch(schema, pq.read_table(m.file_name)) for m in result.after])
    assert got.equals(want), got.first_difference(want)
    assert sum(m.row_count for m in result.after) == want.n_rows
    assert all(m.level == 5 and m.row_count <= 1000 for m in result.after) and len(result.after) >= 4
    for a, b in zip(result.after, result.after[1:]):                 # the output is one sorted run
        assert a.max_key < b.min_key
    kinds = np.asarray(want.columns[schema.n_key + 1].data[: want.n_rows])
    assert sum(m.delete_row_count for m in result.after) == int(np.isin(kinds, [1, 3]).sum())
    if drop_delete:
        assert sum(m.delete_row_count for m in result.after) == 0


@pytest.mark.parametrize("key_kind", ["string", "composite"])
def test_rewritten_files_carry_full_key_bounds(tmp_path, key_kind):
    """min_key / max_key of a compaction's output are the key ROWS of the file's first and last record
    (KeyValueDataFileWriter.java:116-118,166-167) — strings and every field of a composite key — so that the output
    can be fed back into IntervalPartition / key-range pruning / another compaction."""
    from paimon_b200.merge_tree_readers import MergeFileSplitRead, comparable_key
    if key_kind == "string":
        vt = RowType((DataField("pk", "VARCHAR(16)", False), DataField("v", "BIGINT", True), DataField("s", "STRING", True)))
        schema = KeyValueSchema.of(vt, ["pk"])
        def key_of(k): return ("user_%07d" % k,)
    else:
        vt = RowType((DataField("a", "INT", False), DataField("b", "VARCHAR(8)", False), DataField("v", "BIGINT", True),
                      DataField("s", "STRING", True)))
        schema = KeyValueSchema.of(vt, ["a", "b"])
        def key_of(k): return (k // 50, "b%02d" % (k % 50))
    rng = random.Random(3)
    metas, file_runs = [], []
    for f in range(6):
        ks = sorted(rng.sample(range(3000), 900))
        rows = [key_of(k) + (f * 10000 + i, 0) + key_of(k) + (k * 7 + f, None if k % 4 == 0 else "s%d" % k)
                for i, k in enumerate(ks)]
        batch = KeyValueBatch.from_rows(schema, rows)
        path = str(tmp_path / f"in-{f}.parquet")
        write_kv_parquet(batch, path)
        first, last = key_of(ks[0]), key_of(ks[-1])
        metas.append(DataFileMeta(path, 0, batch.n_rows, first[0] if len(first) == 1 else first,
                                  last[0] if len(last) == 1 else last))
        file_runs.append(batch)
    factory = DeduplicateMergeFunction.factory()
    rewriter = MergeTreeCompactRewriter(schema, factory, str(tmp_path), target_file_rows=700, page_rows=128)
    result = rewriter.rewrite_compaction(3, False, IntervalPartition(metas).partition())
    want = pyoracle.merge(schema, factory.create(), file_runs)
    outs = [arrow_to_batch(schema, pq.read_table(m.file_name)) for m in result.after]
    assert concat_batches(schema, outs).equals(want)
    for m, b in zip(result.after, outs):
        rows = b.to_rows()
        lo, hi = rows[0][: schema.n_key], rows[-1][: schema.n_key]
        assert m.min_key == (lo[0] if schema.n_key == 1 else tuple(lo))
        assert m.max_key == (hi[0] if schema.n_key == 1 else tuple(hi))
    for a, b in zip(result.after, result.after[1:]):
        assert comparable_key(a.max_key) < comparable_key(b.min_key)
    # the output re-partitions into ONE section of ONE run, and a key-range read prunes by the bounds
    sections = IntervalPartition(result.after).partition()
    assert len(sections) >= 1 and all(len(sec) == 1 for sec in sections)
    read = MergeFileSplitRead(schema, factory).with_key_filter(result.after[1].min_key, result.after[1].max_key)
    assert [f.file_name for f in read._prune(result.after)] == [result.after[1].file_name]
    # and compacts again to the same rows
    again = MergeTreeCompactRewriter(schema, factory, str(tmp_path / "x"), target_file_rows=100000)
    import os
    os.makedirs(str(tmp_path / "x"))
    res2 = again.rewrite_compaction(4, False, IntervalPartition(result.after).partition())
    got2 = concat_batches(schema, [arrow_to_batch(schema, pq.read_table(m.file_name)) for m in res2.after])
    assert got2.equals(want)
