"""Parquet decode on the device vs pyarrow (the byte-level decode oracle), and the fused decode -> merge
path vs the merge oracle.  Mirrors the reference's round-trip strategy
(paimon-format/src/test/java/org/apache/paimon/format/parquet/ParquetReadWriteTest.java:203-258, 744-816:
row-group sizes {10, 1000}, dictionary on/off, nulls, all supported types)."""
import random

import numpy as np
import pyarrow.parquet as pq
import pytest

from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import KeyValueBatch
from paimon_b200.format import FileFormat, FormatReaderContext, LocalFileIO
from paimon_b200.merge_function import DeduplicateMergeFunction, PartialUpdateMergeFunction
from paimon_b200.sort_merge_reader import SortMergeReader
from paimon_b200.types import DataField, KeyValueSchema, RowType

from parquet_util import arrow_to_batch, write_kv_parquet

pytestmark = pytest.mark.gpu


def decode(schema, path):
    fmt = FileFormat.from_identifier("parquet")
    rd = fmt.create_reader_factory(schema).create_reader(FormatReaderContext(LocalFileIO(), path))
    try:
        batch = rd.read_batch()
        assert rd.read_batch() is None
        return batch, rd.info()
    finally:
        rd.close()


def check_file(schema, batch, path, **opts):
    write_kv_parquet(batch, path, **opts)
    got, info = decode(schema, path)
    want = arrow_to_batch(schema, pq.read_table(path))
    if batch.n_rows == 0:
        assert got is None
        return info
    assert got.equals(want), got.first_difference(want)
    assert got.equals(batch), got.first_difference(batch)
    return info


WRITER_OPTS = [
    dict(),
    dict(use_dictionary=False),
    dict(data_page_version="2.0"),
    dict(data_page_version="2.0", use_dictionary=False),
    dict(row_group_size=10),
    dict(row_group_size=1000, data_page_size=512),
    dict(data_page_size=256, dictionary_pagesize_limit=512),       # dictionary overflow -> PLAIN fallback pages
    dict(compression="snappy"),                                    # Snappy pages are decompressed on the device
    dict(compression="snappy", use_dictionary=False, data_page_version="2.0"),
    dict(compression="snappy", row_group_size=1000, data_page_size=512),
    dict(compression="zstd"),                                      # Paimon's default 'file.compression'
    dict(compression="zstd", compression_level=1, use_dictionary=False),
    dict(compression="zstd", data_page_version="2.0", row_group_size=1000, data_page_size=512),
    dict(compression="gzip"),
    dict(compression="gzip", use_dictionary=False, data_page_version="2.0", data_page_size=4096),
]


@pytest.mark.parametrize("opts", WRITER_OPTS)
def test_wide_row_all_supported_types(tmp_path, opts):
    schema = datagen.schema_c3(n_i64=3, n_f64=2, n_str=3)
    run = datagen.make_runs(schema, 1, 6000, seed=7, null_prob=0.4, delete_prob=0.1)[0]
    info = check_file(schema, run, str(tmp_path / "f.parquet"), **opts)
    assert info.n_rows == run.n_rows and info.launches >= 3


def test_narrow_ints_floats_binary_and_nulls(tmp_path):
    vt = RowType((DataField("pk", "INT", False), DataField("t", "TINYINT", True), DataField("s", "SMALLINT", True),
                  DataField("i", "INT", True), DataField("f", "FLOAT", True), DataField("d", "DOUBLE", True),
                  DataField("str", "STRING", True), DataField("bin", "BINARY", True), DataField("nn", "BIGINT", False)))
    schema = KeyValueSchema.of(vt, ["pk"])
    rng = random.Random(5)
    for n in (0, 1, 31, 32, 33, 1000, 4097):
        rows = []
        for k in range(n):
            def opt(v):
                return None if rng.random() < 0.25 else v
            rows.append((k, k * 3 + 1, rng.choice([0, 1, 2, 3]), k, opt(rng.randrange(-128, 128)),
                         opt(rng.randrange(-32768, 32768)), opt(rng.randrange(-2 ** 31, 2 ** 31)),
                         opt(np.float32(rng.uniform(-1e3, 1e3)).item()), opt(rng.uniform(-1e9, 1e9)),
                         opt("".join(rng.choice("abcdefgh") for _ in range(rng.randrange(0, 40)))),
                         opt(bytes(rng.randrange(256) for _ in range(rng.randrange(0, 20)))), rng.randrange(-10 ** 12, 10 ** 12)))
        batch = KeyValueBatch.from_rows(schema, rows)
        for opts in (dict(), dict(use_dictionary=False, data_page_version="2.0"), dict(row_group_size=100)):
            check_file(schema, batch, str(tmp_path / f"n{n}.parquet"), **opts)


def test_all_null_and_no_null_columns(tmp_path):
    schema = datagen.schema_c2()
    run = datagen.make_runs(schema, 1, 3000, seed=2, null_prob=0.0)[0]
    check_file(schema, run, str(tmp_path / "nonull.parquet"))
    run = datagen.make_runs(schema, 1, 3000, seed=2, null_prob=1.0)[0]
    check_file(schema, run, str(tmp_path / "allnull.parquet"), use_dictionary=False)


def test_large_file_many_pages(tmp_path):
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    run = datagen.make_runs(schema, 1, 600_000, seed=11, null_prob=0.5)[0]
    info = check_file(schema, run, str(tmp_path / "big.parquet"), row_group_size=100_000)
    assert info.n_row_groups == 3 and info.n_data_pages > 3 * schema.n_cols


@pytest.mark.parametrize("engine", ["dedup", "partial-update"])
def test_fused_decode_then_merge_matches_oracle(tmp_path, engine):
    """KeyValueFileReaderFactory -> MergeTreeReaders.readerForSection: files decoded on the device feed the
    merge without a host round trip."""
    schema = datagen.schema_c3(n_i64=3, n_f64=2, n_str=2)
    runs = datagen.make_runs(schema, 6, 60000, seed=21, null_prob=0.5)
    spec = (DeduplicateMergeFunction.factory().create() if engine == "dedup"
            else PartialUpdateMergeFunction.factory({}, schema.value_type, ["pk"]).create())
    fmt = FileFormat.from_identifier("parquet")
    factory = fmt.create_reader_factory(schema)
    file_readers, run_readers = [], []
    for r, run in enumerate(runs):
        path = str(tmp_path / f"run{r}.parquet")
        write_kv_parquet(run, path, use_dictionary=(r % 2 == 0), data_page_version="2.0" if r % 3 == 0 else "1.0")
        fr = factory.create_reader(FormatReaderContext(LocalFileIO(), path))
        file_readers.append(fr)
        run_readers.append(fr.as_sorted_run_reader())
    rd = SortMergeReader.create_sort_merge_reader(run_readers, None, None, spec)
    try:
        rd.execute()
        got = rd.fetch()
    finally:
        rd.close()
        for fr in file_readers:
            fr.close()
    want = pyoracle.merge(schema, spec, runs)
    assert got.equals(want), got.first_difference(want)


def test_unsupported_format_is_refused():
    with pytest.raises(N.UnsupportedOnDevice):
        FileFormat.from_identifier("avro")


def test_unsupported_codec_is_refused(tmp_path):
    """lz4 / brotli pages are not decoded on the device: refused when the file is opened, no CPU fallback."""
    schema = datagen.schema_c2()
    run = datagen.make_runs(schema, 1, 200, seed=2)[0]
    path = str(tmp_path / "z.parquet")
    write_kv_parquet(run, path, compression="lz4")
    with pytest.raises(N.UnsupportedOnDevice):
        decode(schema, path)


def test_snappy_large_pages_and_long_matches(tmp_path):
    """Snappy streams with long literals, long and overlapping copies (runs of equal bytes), several pages."""
    vt = RowType((DataField("pk", "BIGINT", False), DataField("s", "STRING", True), DataField("z", "BIGINT", True)))
    schema = KeyValueSchema.of(vt, ["pk"])
    rows = []
    for k in range(30000):
        text = ("a" * (k % 300)) + ("xyz" * (k % 17)) + str(k * 7919 % 1000003)
        rows.append((k, k, 0, k, None if k % 11 == 0 else text, 0 if k % 3 else k))
    batch = KeyValueBatch.from_rows(schema, rows)
    for opts in (dict(compression="snappy", use_dictionary=False),
                 dict(compression="snappy", use_dictionary=False, data_page_version="2.0", data_page_size=1 << 16),
                 dict(compression="snappy"),
                 dict(compression="zstd", use_dictionary=False),
                 dict(compression="zstd", use_dictionary=False, data_page_version="2.0", data_page_size=1 << 16),
                 dict(compression="zstd", compression_level=9)):
        check_file(schema, batch, str(tmp_path / "snappy.parquet"), **opts)


def test_merge_file_split_read_end_to_end(tmp_path):
    """MergeFileSplitRead.createMergeReader over Parquet data files: IntervalPartition -> sections ->
    per-section device merge -> concat -> drop delete, against the oracle merging every file as its own run
    (CORE-T/operation/MergeFileSplitReadTest: scan result == model of the table)."""
    from paimon_b200.merge_tree_readers import DataFileMeta, IntervalPartition, MergeFileSplitRead, concat_batches
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    rng = np.random.default_rng(42)
    metas, file_runs = [], []
    # three key ranges; inside each, several overlapping files (level 0) and one chain of disjoint files (level 1)
    for sec, (lo, hi) in enumerate([(0, 3000), (5000, 9000), (20000, 20500)]):
        for f in range(4):
            keys = np.sort(rng.choice(np.arange(lo, hi), size=int((hi - lo) * 0.3), replace=False)).astype(np.int64)
            file_runs.append(datagen.make_run(schema, len(file_runs), keys, seed=9, null_prob=0.4, delete_prob=0.1))
        step = (hi - lo) // 3
        for j in range(3):                                   # a sorted run made of three key-disjoint files
            keys = np.arange(lo + j * step, lo + (j + 1) * step - 5, 2, dtype=np.int64)
            file_runs.append(datagen.make_run(schema, len(file_runs), keys, seed=9, null_prob=0.4))
    for i, run in enumerate(file_runs):
        path = str(tmp_path / f"data-{i}.parquet")
        write_kv_parquet(run, path, use_dictionary=(i % 2 == 0))
        k = run.columns[0].data
        metas.append(DataFileMeta(path, 0, run.n_rows, int(k[0]), int(k[-1]), level=0))
    sections = IntervalPartition(metas).partition()
    assert len(sections) == 3 and all(len(s) == 5 for s in sections)       # 4 overlapping files + 1 chain each
    assert sorted(len(r.files) for r in sections[0]) == [1, 1, 1, 1, 3]
    for keep_delete in (False, True):
        spec = PartialUpdateMergeFunction.factory({"ignore-delete": "true"}, schema.value_type, ["pk"])
        read = MergeFileSplitRead(schema, spec)
        rd = read.create_merge_reader(metas, keep_delete=keep_delete)
        batches = []
        while True:
            b = rd.read_batch()
            if b is None:
                break
            batches.append(b)
        rd.close()
        got = concat_batches(schema, batches)
        want = pyoracle.merge(schema, spec.create().with_drop_delete(not keep_delete), file_runs)
        assert got.equals(want), got.first_difference(want)


def _filter_batch(schema, batch, deleted):
    keep = np.ones(batch.n_rows, bool)
    keep[[d for d in deleted if d < batch.n_rows]] = False
    rows = [r for r, k in zip(batch.to_rows(), keep) if k]
    return KeyValueBatch.from_rows(schema, rows)


@pytest.mark.parametrize("n,frac", [(0, 0.0), (1, 1.0), (37, 0.3), (5000, 0.0), (5000, 0.5), (5000, 1.0), (70000, 0.1)])
def test_apply_deletion_vector(n, frac):
    """ApplyDeletionVectorReader: rows whose file position is in the deletion vector disappear
    (paimon-core/.../deletionvectors/ApplyDeletionVectorReader.java:31-54), every column type, nulls kept."""
    from paimon_b200.sort_merge_reader import SortedRunReader, apply_deletion_vector
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    run = datagen.make_runs(schema, 1, 2 * n, seed=13, null_prob=0.3, delete_prob=0.1)[0] if n else \
        KeyValueBatch.from_rows(schema, [])
    rng = np.random.default_rng(n)
    deleted = sorted(rng.choice(run.n_rows, size=int(run.n_rows * frac), replace=False).tolist()) if run.n_rows else []
    rd = SortedRunReader(schema, run)
    out = apply_deletion_vector(schema, rd, deleted + [10 ** 6] if frac not in (0.0, 1.0) else deleted)
    try:
        got = out.read_batch()
    finally:
        out.close()
        rd.close()
    want = _filter_batch(schema, run, deleted)
    if want.n_rows == 0:
        assert got is None or got.n_rows == 0
    else:
        assert got.equals(want), got.first_difference(want)


def test_merge_with_deletion_vectors(tmp_path):
    """KeyValueFileReaderFactory with a DeletionVector.Factory: the merge sees the files minus their deleted rows."""
    from paimon_b200.merge_tree_readers import (DataFileMeta, IntervalPartition, KeyValueFileReaderFactory,
                                                MergeTreeReaders, concat_batches)
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=1)
    runs = datagen.make_runs(schema, 4, 8000, seed=6, null_prob=0.3)
    rng = np.random.default_rng(3)
    metas, dvs, filtered = [], {}, []
    for i, run in enumerate(runs):
        path = str(tmp_path / f"f{i}.parquet")
        write_kv_parquet(run, path)
        k = run.columns[0].data
        metas.append(DataFileMeta(path, 0, run.n_rows, int(k[0]), int(k[-1])))
        dvs[path] = sorted(rng.choice(run.n_rows, size=run.n_rows // (i + 2), replace=False).tolist()) if i != 2 else None
        filtered.append(_filter_batch(schema, run, dvs[path] or []))
    factory = KeyValueFileReaderFactory(schema, dv_factory=lambda name: dvs[name])
    spec = DeduplicateMergeFunction.factory().create()
    sections = IntervalPartition(metas).partition()
    rd = MergeTreeReaders.reader_for_merge_tree(sections, factory, None, spec)
    batches = []
    while True:
        b = rd.read_batch()
        if b is None:
            break
        batches.append(b)
    rd.close()
    got = concat_batches(schema, batches)
    want = pyoracle.merge(schema, spec, filtered)
    assert got.equals(want), got.first_difference(want)


@pytest.mark.parametrize("opts", [dict(), dict(data_page_version="2.0"), dict(data_page_size=2048),
                                  dict(data_page_version="2.0", data_page_size=512, row_group_size=3000)])
def test_delta_binary_packed_integers(tmp_path, opts):
    """DELTA_BINARY_PACKED on the integer columns (what parquet.writer.version=v2 produces;
    VectorizedDeltaBinaryPackedReader.java), PLAIN elsewhere; nulls, negative deltas, several pages."""
    vt = RowType((DataField("pk", "BIGINT", False), DataField("t", "TINYINT", True), DataField("s", "SMALLINT", True),
                  DataField("i", "INT", True), DataField("l", "BIGINT", True), DataField("d", "DOUBLE", True),
                  DataField("str", "STRING", True), DataField("c", "BIGINT", False)))
    schema = KeyValueSchema.of(vt, ["pk"])
    rng = random.Random(91)
    for n in (1, 2, 33, 129, 7000):
        rows = []
        for k in range(n):
            def opt(v):
                return None if rng.random() < 0.2 else v
            rows.append((k * 3, (k * 7919) % 1000 + (1 << 40), rng.choice([0, 3]), k * 3, opt(rng.randrange(-128, 128)),
                         opt(rng.randrange(-32768, 32768)), opt(rng.randrange(-2 ** 31, 2 ** 31)),
                         opt(rng.choice([-2 ** 63, 2 ** 63 - 1, 0, rng.randrange(-10 ** 15, 10 ** 15)])),
                         opt(rng.uniform(-1e6, 1e6)), opt("v%d" % k), 7))
        batch = KeyValueBatch.from_rows(schema, rows)
        enc = {f.name: "DELTA_BINARY_PACKED" for f in schema.file_fields()
               if f.physical.name in ("INT8", "INT16", "INT32", "INT64")}
        enc.update({f.name: "PLAIN" for f in schema.file_fields() if f.name not in enc})
        check_file(schema, batch, str(tmp_path / f"delta{n}.parquet"), use_dictionary=False, column_encoding=enc, **opts)


# ------------------------------------------------------------------ section decode: runs are runs, one launch set

def _fetch_and_close(readers):
    out = []
    for r in readers:
        try:
            out.append(r.read_batch())
        finally:
            r.close()
    return out


def test_section_runs_are_concatenations_of_their_files(tmp_path):
    """pg_parquet_read_section: every file of a section in one batch of launches; the files of a run (key-disjoint,
    in key order) come back as ONE run (MergeTreeReaders.readerForRun's ConcatRecordReader).  Files differ in page
    version, dictionary use, page / row-group size and codec; row counts are not multiples of 32, so validity words
    and var-len offsets continue across file boundaries."""
    from paimon_b200.format import read_section
    from paimon_b200.merge_tree_readers import concat_batches
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=3)
    opts = [dict(), dict(use_dictionary=False), dict(data_page_version="2.0"), dict(compression="snappy"),
            dict(row_group_size=700, data_page_size=512), dict(use_dictionary=False, data_page_version="2.0", data_page_size=300),
            dict(data_page_size=256, dictionary_pagesize_limit=512)]
    rng = np.random.default_rng(5)
    run_sizes = [[1237, 1, 3001, 33], [5], [], [64, 4099]]          # files per run; run 2 is empty
    files, want, key0, fi = [], [], 0, 0
    for r, sizes in enumerate(run_sizes):
        parts = []
        for n in sizes:
            keys = np.arange(key0, key0 + 3 * n, 3, dtype=np.int64)
            key0 += 3 * n + 10
            part = datagen.make_run(schema, fi, keys, seed=3, null_prob=0.35, delete_prob=0.1)
            path = str(tmp_path / f"f{fi}.parquet")
            write_kv_parquet(part, path, **opts[fi % len(opts)])
            files.append((open(path, "rb").read(), r))
            parts.append(arrow_to_batch(schema, pq.read_table(path)))
            fi += 1
        want.append(concat_batches(schema, parts) if parts else None)
    readers, info = read_section(schema, files, len(run_sizes))
    assert info.n_files == len(files) and info.n_runs == len(run_sizes)
    assert info.n_rows == sum(sum(s) for s in run_sizes)
    assert info.launches <= 12                              # per SECTION, not per file
    got = _fetch_and_close(readers)
    for r, (g, w) in enumerate(zip(got, want)):
        if w is None or w.n_rows == 0:
            assert g is None or g.n_rows == 0
        else:
            assert g.equals(w), f"run {r}: " + g.first_difference(w)


def test_section_from_an_asynchronous_upload(tmp_path):
    """pg_files_upload_begin / wait / free: the files of the next section travel to the device on the library's upload
    stream; the descriptors wait() hands back decode to the same runs as the host bytes do."""
    from paimon_b200.format import FileUpload, read_section
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    files, uploads = [], []
    for i, n in enumerate((3001, 17, 1200)):
        keys = np.arange(i * 100_000, i * 100_000 + n, dtype=np.int64)
        part = datagen.make_run(schema, i, keys, seed=9, null_prob=0.4, delete_prob=0.1)
        path = str(tmp_path / f"u{i}.parquet")
        write_kv_parquet(part, path, compression=["zstd", "snappy", "none"][i])
        files.append((open(path, "rb").read(), i % 2))
    files.sort(key=lambda f: f[1])
    want = _fetch_and_close(read_section(schema, files, 2)[0])
    # two uploads in flight, consumed in order
    uploads = [FileUpload(files), FileUpload(files)]
    try:
        for up in uploads:
            dev_files = up.wait()
            assert [r for _, r in dev_files] == [r for _, r in files]
            got = _fetch_and_close(read_section(schema, dev_files, 2)[0])
            for g, w in zip(got, want):
                assert g.equals(w), g.first_difference(w)
    finally:
        for up in uploads:
            up.close()
    with pytest.raises(N.PaimonGpuError):
        N.check(N.load().pg_files_upload_free(12345))


def test_boolean_columns_plain_and_rle(tmp_path):
    """BOOLEAN: PLAIN pages are bit-packed LSB first (VectorizedPlainValuesReader.java:68-84); data page V2 writers
    use RLE for booleans."""
    vt = RowType((DataField("pk", "BIGINT", False), DataField("b", "BOOLEAN", True), DataField("c", "BOOLEAN", False),
                  DataField("s", "STRING", True)))
    schema = KeyValueSchema.of(vt, ["pk"])
    rng = random.Random(8)
    for n in (1, 7, 8, 9, 1000, 20001):
        rows = [(k, k, 0, k, None if rng.random() < 0.3 else rng.random() < 0.5, (k // 37) % 2 == 0,
                 None if k % 5 == 0 else "x" * (k % 9)) for k in range(n)]
        batch = KeyValueBatch.from_rows(schema, rows)
        for opts in (dict(), dict(data_page_version="2.0"), dict(use_dictionary=False, data_page_size=128),
                     dict(data_page_version="2.0", compression="snappy", data_page_size=200)):
            check_file(schema, batch, str(tmp_path / f"bool{n}.parquet"), **opts)


def test_section_from_device_resident_file_images(tmp_path):
    """Files whose bytes already sit in HBM (PG_MEM_DEVICE): the encoder's device image goes straight back into the
    decoder — footers are fetched to the host, page headers are parsed on the device."""
    import ctypes as C
    from paimon_b200.compact_rewriter import file_column_names
    from paimon_b200.format import read_section
    from paimon_b200.merge_tree_readers import concat_batches
    from paimon_b200.sort_merge_reader import SortedRunReader, _SchemaHandle
    schema = datagen.schema_c3(n_i64=3, n_f64=2, n_str=3)
    lib = N.init(0)
    sh = _SchemaHandle(schema, 0)
    names = file_column_names(schema)
    arr = (C.c_char_p * len(names))(*[nm.encode() for nm in names])
    parts, files, handles, rds = [], [], [], []
    try:
        for i, n in enumerate((40000, 1234, 70001)):
            keys = np.arange(i * 1_000_000, i * 1_000_000 + n, dtype=np.int64)
            part = datagen.make_run(schema, i, keys, seed=4, null_prob=0.5, delete_prob=0.05)
            rd = SortedRunReader(schema, part)
            rds.append(rd)
            fh = C.c_uint64(0)
            opts = N.PgParquetWriteOptions(16384, 2000)
            N.check(lib.pg_parquet_encode(rd._open(sh.handle), arr, 0, -1, C.byref(opts), C.byref(fh)))
            handles.append(fh.value)
            ptr, size = C.c_void_p(0), C.c_int64(0)
            N.check(lib.pg_parquet_file_device_image(fh.value, C.byref(ptr), C.byref(size)))
            files.append(((ptr.value, size.value), 0))
            parts.append(part)
            # the patched device image is the same file pg_parquet_file_fetch assembles on the host
            host = np.zeros(size.value, np.uint8)
            N.check(lib.pg_parquet_file_fetch(fh.value, host.ctypes.data, size.value))
            p = str(tmp_path / f"img{i}.parquet")
            host.tofile(p)
            assert arrow_to_batch(schema, pq.read_table(p)).equals(part)
        readers, info = read_section(schema, files, 1)
        got = _fetch_and_close(readers)[0]
        want = concat_batches(schema, parts)
        assert got.equals(want), got.first_difference(want)
        assert info.n_data_pages >= sum(-(-p.n_rows // 2000) for p in parts) * schema.n_cols
    finally:
        for h in handles:
            lib.pg_parquet_file_free(h)
        for rd in rds:
            rd.close()
        sh.close()


def test_wide_fan_in_of_files_is_few_runs(tmp_path):
    """One wide level-0 file over a higher-level run made of 40 small files: 2 merge inputs for the reference
    (IntervalPartition + ConcatRecordReader), and 2 here — not 41 (> PG_MAX_RUNS)."""
    from paimon_b200.merge_tree_readers import DataFileMeta, MergeFileSplitRead, concat_batches
    schema = datagen.schema_c3(n_i64=1, n_f64=1, n_str=1)
    metas, file_runs = [], []
    for j in range(40):
        keys = np.arange(j * 1000, j * 1000 + 900, 2, dtype=np.int64)
        file_runs.append(datagen.make_run(schema, 0, keys, seed=2, null_prob=0.3))
    rng = np.random.default_rng(1)
    keys = np.sort(rng.choice(40000, size=9000, replace=False)).astype(np.int64)
    file_runs.append(datagen.make_run(schema, 1, keys, seed=2, null_prob=0.3, delete_prob=0.1))
    for i, run in enumerate(file_runs):
        path = str(tmp_path / f"d{i}.parquet")
        write_kv_parquet(run, path)
        k = run.columns[0].data
        metas.append(DataFileMeta(path, 0, run.n_rows, int(k[0]), int(k[-1]), level=5 if i < 40 else 0))
    spec = PartialUpdateMergeFunction.factory({"ignore-delete": "true"}, schema.value_type, ["pk"])
    rd = MergeFileSplitRead(schema, spec).create_merge_reader(metas)
    batches = []
    while True:
        b = rd.read_batch()
        if b is None:
            break
        batches.append(b)
    rd.close()
    got = concat_batches(schema, batches)
    want = pyoracle.merge(schema, spec.create().with_drop_delete(True), file_runs)
    assert got.equals(want), got.first_difference(want)


# ------------------------------------------------------------------ read-type projection

def _drain(rd):
    from paimon_b200.merge_tree_readers import concat_batches
    batches = []
    while True:
        b = rd.read_batch()
        if b is None:
            break
        batches.append(b)
    rd.close()
    return batches


@pytest.mark.parametrize("engine", ["dedup", "partial-update", "partial-update-seq", "aggregation"])
def test_read_type_projection_is_pushed_into_decode_and_merge(tmp_path, engine):
    """MergeFileSplitRead.withReadType (MergeFileSplitRead.java:133-163): only the wanted value fields are decoded
    and merged; the result equals the full merge with the other columns removed.  With 'sequence.field' the sequence
    column is still decoded (the merge compares it) although it is not part of the read type."""
    from paimon_b200.merge_function import AggregateMergeFunction
    from paimon_b200.merge_tree_readers import DataFileMeta, MergeFileSplitRead
    schema = datagen.schema_c3(n_i64=4, n_f64=3, n_str=3)
    runs = datagen.make_runs(schema, 5, 40000, seed=77, null_prob=0.4)
    metas = []
    for i, run in enumerate(runs):
        path = str(tmp_path / f"p{i}.parquet")
        write_kv_parquet(run, path, use_dictionary=(i % 2 == 0), compression="zstd" if i == 3 else "none")
        k = run.columns[0].data
        metas.append(DataFileMeta(path, 0, run.n_rows, int(k[0]), int(k[-1])))
    vt = schema.value_type
    if engine == "dedup":
        factory, udsc = DeduplicateMergeFunction.factory(), None
    elif engine == "partial-update":
        factory, udsc = PartialUpdateMergeFunction.factory({}, vt, ["pk"]), None
    elif engine == "partial-update-seq":
        from paimon_b200.merge_function import UserDefinedSeqComparator
        opts = {"sequence.field": "i0"}
        factory, udsc = PartialUpdateMergeFunction.factory(opts, vt, ["pk"]), UserDefinedSeqComparator.create(vt, opts)
    else:
        factory, udsc = AggregateMergeFunction.factory({"fields.i1.aggregate-function": "sum",
                                                        "fields.d2.aggregate-function": "max"}, vt, ["pk"]), None
    wanted = ["pk", "i1", "d2", "s0"]
    mask = [n in wanted for n in vt.field_names()]
    read = MergeFileSplitRead(schema, factory, udsc).with_read_type(wanted)
    batches = _drain(read.create_merge_reader(metas, keep_delete=True))
    assert len(batches) == 1
    got = batches[0]
    spec = factory.create()
    if udsc is not None:
        spec = udsc.apply(spec.normalised(schema.n_val))
    want = pyoracle.merge(schema, spec, runs).project(mask)
    assert [c is None for c in got.columns] == [c is None for c in want.columns]
    assert got.equals(want), got.first_difference(want)
    # the projection alone, on host runs (no files): the merge emits the read type only
    from paimon_b200.sort_merge_reader import merge_runs
    got2 = merge_runs(schema, spec.with_read_fields(mask), runs)
    assert got2.equals(want), got2.first_difference(want)


@pytest.mark.parametrize("engine", ["dedup", "dedup-ignore-delete", "first-row", "partial-update"])
def test_section_with_more_than_32_sorted_runs(tmp_path, engine):
    """70 overlapping files = 70 sorted runs in one section (MergeSorter.java:112-198 merges any number at once):
    merged in rounds of 32 on the device where that is exact (deduplicate, first-row), refused for merge functions
    that fold all records of a key in sequence order."""
    from paimon_b200.merge_function import FirstRowMergeFunction
    from paimon_b200.merge_tree_readers import DataFileMeta, MergeFileSplitRead, concat_batches
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=1)
    rng = np.random.default_rng(12)
    metas, file_runs = [], []
    for i in range(70):
        keys = np.sort(rng.choice(20000, size=1500, replace=False)).astype(np.int64)
        run = datagen.make_run(schema, i, keys, seed=8, null_prob=0.3, delete_prob=0.0 if engine == "first-row" else 0.1)
        path = str(tmp_path / f"o{i}.parquet")
        write_kv_parquet(run, path)
        metas.append(DataFileMeta(path, 0, run.n_rows, int(keys[0]), int(keys[-1])))
        file_runs.append(run)
    factory = {"dedup": DeduplicateMergeFunction.factory(),
               "dedup-ignore-delete": DeduplicateMergeFunction.factory({"ignore-delete": "true"}),
               "first-row": FirstRowMergeFunction.factory({}),
               "partial-update": PartialUpdateMergeFunction.factory({"ignore-delete": "true"}, schema.value_type, ["pk"])}[engine]
    read = MergeFileSplitRead(schema, factory)
    if engine == "partial-update":
        with pytest.raises(N.UnsupportedOnDevice, match="32 sorted runs"):
            read.create_merge_reader(metas).read_batch()
        return
    got = concat_batches(schema, _drain(read.create_merge_reader(metas)))
    want = pyoracle.merge(schema, factory.create().with_drop_delete(True), file_runs)
    assert got.equals(want), got.first_difference(want)
