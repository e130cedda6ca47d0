"""The bloom-filter file index built on the device (pg_bloom_filter_build, file_index.py): every filter of every file is
byte-identical to the independent model in file_index_reference.py over exactly the rows of that file, and every
non-NULL value of the file tests positive through the restated FileIndexFormat / BloomFilterFileIndex readers."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import file_index_reference as R
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import Column, KeyValueBatch
from paimon_b200.compact_rewriter import KeyValueDataFileWriter, MergeTreeCompactRewriter, RollingFileWriter
from paimon_b200.file_index import FileIndexOptions
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.merge_tree_readers import DataFileMeta, IntervalPartition
from paimon_b200.sort_merge_reader import SortedRunReader, SortMergeReader, _SchemaHandle
from paimon_b200.types import DataField, KeyValueSchema, PhysicalType, RowType

from parquet_util import write_kv_parquet

pytestmark = pytest.mark.gpu

INDEXED = [("t", "TINYINT"), ("s", "SMALLINT"), ("i", "INT"), ("l", "BIGINT"), ("f", "FLOAT"), ("d", "DOUBLE"),
           ("dt", "DATE"), ("tm", "TIME"), ("ts3", "TIMESTAMP(3)"), ("ts6", "TIMESTAMP(6)"), ("str", "STRING"),
           ("vc", "VARCHAR(40)"), ("ch", "CHAR(5)"), ("bin", "BINARY(6)"), ("vb", "VARBINARY(50)")]
F32_SPECIAL = [0x7FC00000, 0x7FC00001, 0xFFC00000, 0x7F800001, 0xFFFFFFFF, 0x80000000, 0, 0x7F800000, 0xFF800000]
F64_SPECIAL = [0x7FF8000000000000, 0x7FF8000000000001, 0xFFF8000000000000, 0x7FF0000000000001, 1 << 63, 0,
               0x7FF0000000000000, 0xFFF0000000000000]


def all_types_schema():
    return KeyValueSchema.of(RowType(tuple([DataField("pk", "BIGINT", False)] +
                                           [DataField(n, t, True) for n, t in INDEXED])), ["pk"])


def random_values(rng, logical, n, null_p=0.2):
    """(model values, Column): None = NULL; FLOAT / DOUBLE as ('bits', raw bits), NaN payloads and both zeros among
    them; timestamps and dates before 1970 among the integers."""
    root = logical.split("(")[0]
    out = []
    for _ in range(n):
        if rng.random() < null_p:
            out.append(None)
        elif root in ("TINYINT", "SMALLINT", "INT", "BIGINT", "DATE", "TIME", "TIMESTAMP"):
            bits = {"TINYINT": 8, "SMALLINT": 16, "BIGINT": 64, "TIMESTAMP": 64}.get(root, 32)
            lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
            out.append(rng.choice([lo, hi, -1, 0, rng.randrange(-1000, 1000), rng.randrange(lo, hi + 1),
                                   -86_400_000 * 365 * 30 - 123]) if root != "TIMESTAMP"
                       else rng.choice([lo, hi, -1, 0, -1_000_000_000_123, rng.randrange(lo, hi + 1)]))
            out[-1] = max(lo, min(hi, out[-1]))
        elif root == "FLOAT":
            out.append(("bits", rng.choice(F32_SPECIAL + [rng.randrange(1 << 32)])))
        elif root == "DOUBLE":
            out.append(("bits", rng.choice(F64_SPECIAL + [rng.randrange(1 << 64)])))
        elif root in ("STRING", "VARCHAR", "CHAR"):
            longest = {"CHAR": 5, "VARCHAR": 40}.get(root, 44)
            out.append("".join(rng.choice("abcé日xyz") for _ in range(rng.randrange(0, longest + 1))))
        else:
            out.append(bytes(rng.randrange(256) for _ in range(rng.randrange(0, 70))))
    return out


def column_of(logical, values):
    from paimon_b200.types import physical_type
    t = physical_type(logical)
    if t in (PhysicalType.FLOAT, PhysicalType.DOUBLE):
        it = PhysicalType.INT32 if t == PhysicalType.FLOAT else PhysicalType.INT64
        width = 32 if t == PhysicalType.FLOAT else 64
        raw = [None if v is None else R.s64(v[1]) if width == 64 else R.s32(v[1]) for v in values]
        c = Column.from_pylist(it, raw)
        return Column(t, c.data.view(np.float32 if width == 32 else np.float64), None, c.valid)
    return Column.from_pylist(t, values)


def all_types_batch(rng, n):
    schema = all_types_schema()
    values = {name: random_values(rng, logical, n) for name, logical in INDEXED}
    cols = [Column.from_pylist(PhysicalType.INT64, list(range(n))), Column.from_pylist(PhysicalType.INT64, list(range(n))),
            Column.from_pylist(PhysicalType.INT8, [rng.choice([0, 1, 2, 3]) for _ in range(n)]),
            Column.from_pylist(PhysicalType.INT64, list(range(n)))]
    cols += [column_of(logical, values[name]) for name, logical in INDEXED]
    return schema, KeyValueBatch(schema, cols), values


def index_options(columns, items=None, threshold=None):
    o = {"file-index.bloom-filter.columns": ",".join(columns)}
    if items:
        o.update({f"file-index.bloom-filter.{c}.items": str(items) for c in columns})
    if threshold is not None:
        o["file-index.in-manifest-threshold"] = threshold
    return FileIndexOptions.from_options(o)


def index_bytes(meta: DataFileMeta) -> bytes:
    if meta.embedded_index is not None:
        assert meta.extra_files == []
        return meta.embedded_index
    assert meta.extra_files == [meta.file_name + ".index"]
    return open(meta.extra_files[0], "rb").read()


def check_file(meta, logical_of, values_of, items=None):
    """The file's index holds, per column, the model's filter over `values_of[column]`, and every non-NULL value
    tests positive."""
    read = R.read_container(index_bytes(meta))
    assert sorted(c for c, _ in read) == sorted(values_of)
    for col, idx in read:
        assert list(idx) == ["bloom-filter"]
        kw = {"items": items} if items else {}
        assert idx["bloom-filter"] == R.filter_of(logical_of[col], values_of[col], **kw), col
        f = R.BloomFilter.from_bytes(idx["bloom-filter"])
        assert all(f.test_hash(R.fast_hash(logical_of[col], v)) for v in values_of[col] if v is not None)


@pytest.mark.parametrize("fmt", ["parquet", "orc"])
@pytest.mark.parametrize("row0,n_rows", [(0, -1), (16, 301), (8, 5)])
def test_every_indexed_type_from_a_run_handle(tmp_path, fmt, row0, n_rows):
    rng = random.Random(row0 * 7 + n_rows)
    schema, batch, values = all_types_batch(rng, 600)
    if fmt == "orc":            # the ORC encoder does not write TIMESTAMP or CHAR
        names = [n for n, t in INDEXED if not t.startswith(("TIMESTAMP", "CHAR"))]
        schema = KeyValueSchema.of(RowType(tuple([DataField("pk", "BIGINT", False)] +
                                                 [DataField(n, t, True) for n, t in INDEXED if n in names])), ["pk"])
        keep = [0, 1, 2, 3] + [4 + i for i, (n, _) in enumerate(INDEXED) if n in names]
        batch = KeyValueBatch(schema, [batch.columns[i] for i in keep])
    else:
        names = [n for n, _ in INDEXED]
    logical = dict(INDEXED)
    end = 600 if n_rows < 0 else row0 + n_rows
    N.init(0)
    sh = _SchemaHandle(schema, 0)
    rd = SortedRunReader(schema, batch)
    try:
        h = rd._open(sh.handle)
        for items, threshold in ((100, "1 mb"), (None, None)):
            opts = index_options(names, items, threshold)
            w = KeyValueDataFileWriter(schema, str(tmp_path / f"f-{items}.{fmt}"), 1, file_format=fmt, file_index=opts)
            written = w.write(h, row0, n_rows)
            assert (written.meta.embedded_index is not None) == (items == 100)
            check_file(written.meta, logical, {n: values[n][row0:end] for n in names}, items)
    finally:
        rd.close()
        sh.close()


def test_c_abi_refusals_on_a_handle():
    vt = RowType((DataField("pk", "BIGINT", False), DataField("b", "BOOLEAN", True), DataField("v", "BIGINT", True)))
    schema = KeyValueSchema.of(vt, ["pk"])
    batch = KeyValueBatch.from_rows(schema, [(k, k, 0, k, k % 2 == 0, k) for k in range(40)])
    lib = N.init(0)
    sh = _SchemaHandle(schema, 0)
    rd = SortedRunReader(schema, batch)
    try:
        h = rd._open(sh.handle)
        buf = np.zeros(64, np.uint8)
        outs = (C.c_void_p * 1)(buf.ctypes.data)

        def build(column, row0=0, n_rows=-1, items=100, cap=64):
            spec = N.PgBloomFilterSpec(column, items, 0.1)
            return lib.pg_bloom_filter_build(h, row0, n_rows, 1, C.byref(spec), outs, (C.c_int64 * 1)(cap))
        assert build(4) == 2 and b"BOOLEAN" in lib.pg_last_error()
        assert build(5, row0=3) == 1 and b"multiple of 8" in lib.pg_last_error()
        assert build(5, row0=8, n_rows=40) == 1
        assert build(9) == 1 and b"out of range" in lib.pg_last_error()
        assert build(5, cap=63) == 1 and b"needs 64" in lib.pg_last_error()
        assert build(5) == 0
        assert buf.tobytes() == R.filter_of("BIGINT", list(range(40)), items=100)
        assert build(5, row0=40, n_rows=0) == 0                     # no rows: the filter of no value, not nothing
        assert buf.tobytes() == R.filter_of("BIGINT", [], items=100) == bytes([0, 0, 0, 3]) + bytes(60)
    finally:
        rd.close()
        sh.close()


@pytest.mark.parametrize("fmt", ["parquet", "orc"])
@pytest.mark.parametrize("drop_delete", [True, False])
def test_rolling_files_of_a_merged_batch(tmp_path, fmt, drop_delete):
    """A merged batch (retracts kept or dropped) cut into files: each file's index is the model's over its own rows."""
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=1)
    runs = datagen.make_runs(schema, 4, 20000, seed=5, null_prob=0.3, delete_prob=0.2)
    spec = DeduplicateMergeFunction.factory().create().with_drop_delete(drop_delete)
    names = ["i0", "d0", "s0"]
    logical = {"i0": "BIGINT", "d0": "DOUBLE", "s0": "VARCHAR(24)"}
    rd = SortMergeReader.create_sort_merge_reader([SortedRunReader(schema, b) for b in runs], None, None, spec)
    try:
        rd.execute()
        merged = rd.fetch()
        kinds = merged.value_kinds
        assert drop_delete == (not np.isin(kinds, [1, 3]).any())
        rolling = RollingFileWriter(schema, str(tmp_path), 2, 3000, file_format=fmt,
                                    file_index=index_options(names, items=2000, threshold="64 b"))
        files = rolling.write(rd._merge_h, merged.n_rows)
    finally:
        rd.close()
    assert len(files) > 2
    v = {n: merged.value_column(schema.value_type.index_of(n)).to_pylist() for n in names}
    v["d0"] = [None if x is None else ("bits", int(np.float64(x).view(np.uint64))) for x in v["d0"]]
    r0 = 0
    for w in files:
        m = w.meta
        assert m.extra_files == [m.file_name + ".index"] and os.path.exists(m.extra_files[0])
        check_file(m, logical, {n: v[n][r0:r0 + m.row_count] for n in names}, items=2000)
        r0 += m.row_count
    assert r0 == merged.n_rows


def test_compact_rewriter_indexes_every_file(tmp_path):
    schema = datagen.schema_c3(n_i64=1, n_f64=1, n_str=1)
    rng = np.random.default_rng(3)
    metas = []
    for i in range(4):
        keys = np.sort(rng.choice(np.arange(0, 6000), size=2500, replace=False)).astype(np.int64)
        run = datagen.make_run(schema, i, keys, seed=3, null_prob=0.3, delete_prob=0.1)
        path = str(tmp_path / f"in-{i}.parquet")
        write_kv_parquet(run, path)
        metas.append(DataFileMeta(path, 0, run.n_rows, int(keys[0]), int(keys[-1]), level=0))
    options = {"file.format": "orc", "file.compression": "zstd", "file-index.bloom-filter.columns": "s0,i0",
               "file-index.bloom-filter.s0.items": "500", "file-index.bloom-filter.i0.items": "500",
               "file-index.in-manifest-threshold": "300 b"}
    out = tmp_path / "out"
    out.mkdir()
    rewriter = MergeTreeCompactRewriter(schema, DeduplicateMergeFunction.factory(), str(out), target_file_rows=2000,
                                        options=options)
    result = rewriter.rewrite_compaction(3, False, IntervalPartition(metas).partition())
    assert len(result.after) > 1
    from paimon_b200.format import FileFormat, FormatReaderContext, LocalFileIO
    for m in result.after:
        fr = FileFormat.from_identifier("orc").create_reader_factory(schema).create_reader(
            FormatReaderContext(LocalFileIO(), m.file_name))
        try:
            b = fr.read_batch()
        finally:
            fr.close()
        v = {n: b.value_column(schema.value_type.index_of(n)).to_pylist() for n in ("s0", "i0")}
        assert m.embedded_index is None and m.extra_files == [m.file_name + ".index"]   # two 304-byte filters > 300 bytes
        check_file(m, {"s0": "VARCHAR(24)", "i0": "BIGINT"}, v, items=500)
    # without file-index options nothing is indexed
    plain = MergeTreeCompactRewriter(schema, DeduplicateMergeFunction.factory(), str(out), target_file_rows=2000,
                                     options={"file.format": "orc"})
    for m in plain.rewrite_compaction(4, False, IntervalPartition(metas).partition()).after:
        assert m.embedded_index is None and m.extra_files == []
        assert not os.path.exists(m.file_name + ".index")
