"""The decoded runs of a section: the Parquet and the ORC decoder lay out the same runs from the same rows (read columns,
NULL rows of a field some files lack, absent unread columns, `decoded_bytes`), both resolve the files' columns against
the read schema by the same rule, and a deletion vector applied to a projected run keeps the projection."""
import ctypes as C
import random

import numpy as np
import pyarrow.orc as orc
import pyarrow.parquet as pq
import pytest

from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import KeyValueBatch
from paimon_b200.format import read_section
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.merge_tree_readers import concat_batches
from paimon_b200.sort_merge_reader import _SchemaHandle, apply_deletion_vector
from paimon_b200.types import DataField, KeyValueSchema, RowType, is_varlen

from parquet_util import to_arrow

pytestmark = pytest.mark.gpu

VT = RowType((DataField("pk", "BIGINT", False), DataField("a", "BIGINT", True), DataField("i", "INT", True),
              DataField("s", "STRING", True), DataField("t", "STRING", True), DataField("d", "DOUBLE", True)))
SCHEMA = KeyValueSchema.of(VT, ["pk"])
OLD = KeyValueSchema.of(RowType(tuple(f for f in VT.fields if f.name != "a")), ["pk"])    # written before ADD COLUMN a
MASK = [n not in ("i", "t") for n in VT.field_names()]        # drops a fixed-width and a var-len field
RUN_FILES = [[1237, 2003], [515, 3001], []]                   # rows per file; run 2 is empty; file 0 lacks `a`


def _write(batch, path, fmt):
    t = to_arrow(batch)
    if fmt == "parquet":
        pq.write_table(t, path, compression="none")
    else:
        orc.write_table(t, path, compression="zstd")


def _section(tmp_path, fmt):
    """Files of RUN_FILES in `fmt`, as read_section takes them, and the full rows each run must decode to."""
    rng = np.random.default_rng(17)
    files, want, key0 = [], [], 0
    for r, sizes in enumerate(RUN_FILES):
        rows = []
        for n in sizes:
            fi = len(files)
            part = []
            for k in range(key0, key0 + 3 * n, 3):
                def opt(v):
                    return None if rng.random() < 0.3 else v
                part.append((k, k + 100, 0, k, opt(int(rng.integers(-2 ** 62, 2 ** 62))), opt(int(rng.integers(-2 ** 31, 2 ** 31))),
                             opt("s%d" % k), opt("t" * int(rng.integers(0, 20))), opt(float(rng.uniform(-1e6, 1e6)))))
            key0 += 3 * n + 10
            if fi == 0:
                batch = KeyValueBatch.from_rows(OLD, [p[:4] + p[5:] for p in part])
                part = [p[:4] + (None,) + p[5:] for p in part]
            else:
                batch = KeyValueBatch.from_rows(SCHEMA, part)
            path = str(tmp_path / f"f{fi}.{fmt}")
            _write(batch, path, fmt)
            files.append((open(path, "rb").read(), r))
            rows += part
        want.append(KeyValueBatch.from_rows(SCHEMA, rows))
    return files, want


def _layout(handle):
    n = C.c_int64(0)
    data_bytes = np.zeros(SCHEMA.n_cols, np.int64)
    has_valid = np.zeros(SCHEMA.n_cols, np.int32)
    N.check(N.load().pg_run_layout(handle, C.byref(n), data_bytes.ctypes.data, has_valid.ctypes.data, SCHEMA.n_cols))
    return n.value, data_bytes, has_valid


def _filter(batch, deleted):
    gone = set(deleted)
    return KeyValueBatch.from_rows(batch.schema, [row for i, row in enumerate(batch.to_rows()) if i not in gone])


def _fetch_and_close(readers):
    out = []
    for r in readers:
        try:
            out.append(r.read_batch())
        finally:
            r.close()
    return out


def _blob(tmp_path, name, batch, fmt):
    path = str(tmp_path / f"{name}.{fmt}")
    _write(batch, path, fmt)
    return open(path, "rb").read()


@pytest.mark.parametrize("fmt", ["parquet", "orc"])
def test_section_of_empty_files(tmp_path, fmt):
    schema = datagen.schema_c3(n_i64=1, n_f64=1, n_str=1)
    blob = _blob(tmp_path, "empty", KeyValueBatch.from_rows(schema, []), fmt)
    readers, info = read_section(schema, [(blob, 0), (blob, 1)], 2, file_format=fmt)
    assert info.n_rows == 0
    for b in _fetch_and_close(readers):
        assert b is None or b.n_rows == 0


@pytest.mark.parametrize("fmt", ["parquet", "orc"])
def test_columns_are_resolved_by_name_not_position(tmp_path, fmt):
    """The reference resolves file columns by NAME (ParquetReaderFactory.clipParquetSchema): a read schema that lists
    the value fields in another order gets every field's own values — never the positional neighbour's."""
    vt_a = RowType((DataField("pk", "BIGINT", False), DataField("a", "BIGINT", True), DataField("b", "BIGINT", True)))
    vt_b = RowType((DataField("pk", "BIGINT", False), DataField("b", "BIGINT", True), DataField("a", "BIGINT", True)))
    sa, sb = KeyValueSchema.of(vt_a, ["pk"]), KeyValueSchema.of(vt_b, ["pk"])
    batch = KeyValueBatch.from_rows(sa, [(k, k, 0, k, k * 2, k * 3) for k in range(100)])
    blob = _blob(tmp_path, "a", batch, fmt)
    readers, _ = read_section(sa, [(blob, 0)], 1, file_format=fmt)
    assert _fetch_and_close(readers)[0].equals(batch)
    readers, _ = read_section(sb, [(blob, 0)], 1, file_format=fmt)
    swapped = KeyValueBatch.from_rows(sb, [(k, k, 0, k, k * 3, k * 2) for k in range(100)])
    assert _fetch_and_close(readers)[0].equals(swapped)
    # positional reading (no names) of a file whose types line up is what the single-file reader does
    readers, _ = read_section(sb, [(blob, 0)], 1, check_names=False, file_format=fmt)
    assert _fetch_and_close(readers)[0].equals(KeyValueBatch.from_rows(sb, [(k, k, 0, k, k * 2, k * 3) for k in range(100)]))


@pytest.mark.parametrize("fmt", ["parquet", "orc"])
def test_schema_evolution_columns_resolve_by_name(tmp_path, fmt):
    """Files written under older table schemas (ParquetReaderFactory.clipParquetSchema resolves by NAME;
    DataFileRecordReader.java:55-57 casts): an added column is NULL in old files, a dropped column is ignored, column
    order does not matter, INT widened to BIGINT and FLOAT to DOUBLE are cast on the fly."""
    read_vt = RowType((DataField("pk", "BIGINT", False), DataField("a", "BIGINT", True), DataField("f", "DOUBLE", True),
                       DataField("b", "STRING", True), DataField("c", "DOUBLE", True)))
    read_schema = KeyValueSchema.of(read_vt, ["pk"])
    # v1: a INT, f FLOAT, b, no c, plus a column z that was dropped later; v2: another column order
    v1 = KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("z", "INT", True), DataField("a", "INT", True),
                                    DataField("f", "FLOAT", True), DataField("b", "STRING", True))), ["pk"])
    v2 = KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("c", "DOUBLE", True), DataField("b", "STRING", True),
                                    DataField("a", "BIGINT", True), DataField("f", "DOUBLE", True))), ["pk"])
    rng = random.Random(4)

    def opt(v):
        return None if rng.random() < 0.3 else v
    rows1 = [(k, k, 0, k, opt(k * 3), opt(rng.randrange(-2 ** 31, 2 ** 31)), opt(np.float32(rng.uniform(-9, 9)).item()),
              opt("s%d" % k)) for k in range(0, 3000)]
    rows2 = [(k, k, 0, k, opt(k / 7.0), opt("t%d" % k), opt(rng.randrange(-2 ** 62, 2 ** 62)), opt(rng.uniform(-1e9, 1e9)))
             for k in range(5000, 9001)]
    b1 = _blob(tmp_path, "v1", KeyValueBatch.from_rows(v1, rows1), fmt)
    b2 = _blob(tmp_path, "v2", KeyValueBatch.from_rows(v2, rows2), fmt)
    want1 = KeyValueBatch.from_rows(read_schema, [(r[0], r[1], r[2], r[3], r[5], r[6], r[7], None) for r in rows1])
    want2 = KeyValueBatch.from_rows(read_schema, [(r[0], r[1], r[2], r[3], r[6], r[7], r[5], r[4]) for r in rows2])
    # each file as its own run, and both files as ONE run (a fixed-width column that only some files have)
    readers, _ = read_section(read_schema, [(b1, 0), (b2, 1)], 2, file_format=fmt)
    g1, g2 = _fetch_and_close(readers)
    assert g1.equals(want1), g1.first_difference(want1)
    assert g2.equals(want2), g2.first_difference(want2)
    # in ONE run: column c exists in the second file only — allowed for fixed-width columns
    readers, _ = read_section(read_schema, [(b1, 0), (b2, 0)], 1, file_format=fmt)
    both = _fetch_and_close(readers)[0]
    want = concat_batches(read_schema, [want1, want2])
    assert both.equals(want), both.first_difference(want)
    # a NOT NULL read field the file lacks, or a narrowing, is refused
    bad_vt = RowType((DataField("pk", "BIGINT", False), DataField("a", "INT", True), DataField("nn", "BIGINT", False)))
    with pytest.raises(N.UnsupportedOnDevice):
        read_section(KeyValueSchema.of(bad_vt, ["pk"]), [(b2, 0)], 1, file_format=fmt)


WITH_T = KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("a", "BIGINT", True),
                                    DataField("t", "STRING", True))), ["pk"])
NO_T = KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("a", "BIGINT", True))), ["pk"])


def _rows(k0, n, with_t):
    return [(k, k, 0, k, None if k % 3 == 0 else k * 5) + ((None if k % 4 == 0 else "t" * (k % 11),) if with_t else ())
            for k in range(k0, k0 + n)]


@pytest.mark.parametrize("fmt", ["parquet", "orc"])
def test_var_len_column_in_some_files_of_a_run(tmp_path, fmt):
    """A run is judged by its files with rows: a file without rows has no rows to fill, whether or not it has a var-len
    column.  Only a var-len column that some files with rows of the run have and others lack is refused."""
    empty_t = _blob(tmp_path, "empty_t", KeyValueBatch.from_rows(WITH_T, []), fmt)
    empty_no_t = _blob(tmp_path, "empty_no_t", KeyValueBatch.from_rows(NO_T, []), fmt)
    no_t = _blob(tmp_path, "no_t", KeyValueBatch.from_rows(NO_T, _rows(0, 2345, False)), fmt)
    has_t = _blob(tmp_path, "has_t", KeyValueBatch.from_rows(WITH_T, _rows(3000, 1717, True)), fmt)
    # (a) the file with rows lacks t, the empty file has it: t is NULL in every row
    readers, _ = read_section(WITH_T, [(no_t, 0), (empty_t, 0)], 1, file_format=fmt)
    got = _fetch_and_close(readers)[0]
    want = KeyValueBatch.from_rows(WITH_T, [r + (None,) for r in _rows(0, 2345, False)])
    assert got.equals(want), got.first_difference(want)
    # (b) the file with rows has t, the empty file lacks it
    readers, _ = read_section(WITH_T, [(has_t, 0), (empty_no_t, 0)], 1, file_format=fmt)
    got = _fetch_and_close(readers)[0]
    want = KeyValueBatch.from_rows(WITH_T, _rows(3000, 1717, True))
    assert got.equals(want), got.first_difference(want)
    # (c) two files with rows, one of them without t
    with pytest.raises(N.UnsupportedOnDevice):
        read_section(WITH_T, [(no_t, 0), (has_t, 0)], 1, file_format=fmt)


@pytest.mark.parametrize("fmt", ["parquet", "orc"])
def test_null_column_name_and_positional_column_count(tmp_path, fmt):
    """A NULL entry in column_names is an invalid argument; a positional read needs the read schema's column count."""
    has_t = _blob(tmp_path, "has_t", KeyValueBatch.from_rows(WITH_T, _rows(0, 100, True)), fmt)
    with pytest.raises(N.UnsupportedOnDevice):
        read_section(NO_T, [(has_t, 0)], 1, check_names=False, file_format=fmt)
    lib = N.init(0)
    sh = _SchemaHandle(WITH_T, 0)
    try:
        arr = np.frombuffer(has_t, np.uint8)
        files = (N.PgFileDesc * 1)(N.PgFileDesc(arr.ctypes.data, len(arr), N.PG_MEM_HOST, 0))
        nm = [f.name.encode() for f in WITH_T.file_fields()]
        nm[-1] = None
        names = (C.c_char_p * len(nm))(*nm)
        runs = (C.c_uint64 * 1)()
        fn = lib.pg_parquet_read_section if fmt == "parquet" else lib.pg_orc_read_section
        assert fn(sh.handle, files, 1, 1, names, None, runs, None) == 1
        assert b"NULL" in lib.pg_last_error()
    finally:
        sh.close()


def test_parquet_and_orc_build_the_same_runs(tmp_path):
    types = SCHEMA.physical_types()
    got, layouts = {}, {}
    for fmt in ("parquet", "orc"):
        files, want = _section(tmp_path, fmt)
        readers, info = read_section(SCHEMA, files, len(RUN_FILES), read_value_fields=MASK, file_format=fmt)
        try:
            layouts[fmt] = [_layout(rd._handle) for rd in readers]
            got[fmt] = [rd.read_batch() for rd in readers]
        finally:
            for rd in readers:
                rd.close()
        expected = 0
        for n, data_bytes, has_valid in layouts[fmt]:
            for c, t in enumerate(types):
                if data_bytes[c] < 0:
                    continue
                expected += int(data_bytes[c]) + (4 * (n + 1) if is_varlen(t) else 0) + ((n + 7) // 8 if has_valid[c] else 0)
        assert info.decoded_bytes == expected, fmt
        assert info.n_runs == len(RUN_FILES) and info.n_rows == sum(map(sum, RUN_FILES))
        for r, w in enumerate(want):
            w = w.project(MASK)
            if w.n_rows == 0:
                assert got[fmt][r] is None or got[fmt][r].n_rows == 0
            else:
                assert got[fmt][r].equals(w), (fmt, r, got[fmt][r].first_difference(w))
    nk = SCHEMA.n_key + 2
    for g_p, g_o in zip(got["parquet"], got["orc"]):
        assert (g_p is None) == (g_o is None) and (g_p is None or g_p.equals(g_o))
    for (n_p, db_p, _), (n_o, db_o, _) in zip(layouts["parquet"], layouts["orc"]):
        assert n_p == n_o
        assert db_p.tolist() == db_o.tolist()
        assert [db_p[nk + j] < 0 for j in range(len(MASK))] == [not m for m in MASK]


@pytest.mark.parametrize("fmt", ["parquet", "orc"])
def test_deletion_vector_on_a_projected_run(tmp_path, fmt):
    files, want = _section(tmp_path, fmt)
    readers, _ = read_section(SCHEMA, files, len(RUN_FILES), read_value_fields=MASK, file_format=fmt)
    rng = np.random.default_rng(5)
    try:
        for r, rd in enumerate(readers):
            n = want[r].n_rows
            deleted = sorted(rng.choice(n, size=n // 3, replace=False).tolist()) if n else []
            out = apply_deletion_vector(SCHEMA, rd, deleted)
            try:
                _, data_bytes, _ = _layout(out._handle)
                got = out.read_batch()
            finally:
                out.close()
            assert [data_bytes[SCHEMA.n_key + 2 + j] < 0 for j in range(len(MASK))] == [not m for m in MASK]
            w = _filter(want[r], deleted).project(MASK)
            if w.n_rows == 0:
                assert got is None or got.n_rows == 0
            else:
                assert got.equals(w), got.first_difference(w)
    finally:
        for rd in readers:
            rd.close()


@pytest.mark.parametrize("fmt", ["parquet", "orc"])
def test_merge_of_projected_runs_with_deletion_vectors(tmp_path, fmt):
    """MergeTreeReaders.reader_for_section with a read type and a DeletionVector.Factory: the decoder reads the
    projected columns only, and the deletion vectors apply to those runs."""
    from paimon_b200.merge_tree_readers import DataFileMeta, IntervalPartition, KeyValueFileReaderFactory, MergeTreeReaders
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    mask = [n not in ("i1", "s1") for n in schema.value_type.field_names()]
    runs = datagen.make_runs(schema, 4, 6000, seed=8, null_prob=0.3)
    rng = np.random.default_rng(9)
    metas, dvs, filtered = [], {}, []
    for i, run in enumerate(runs):
        path = str(tmp_path / f"m{i}.{fmt}")
        _write(run, path, fmt)
        k = run.columns[0].data
        metas.append(DataFileMeta(path, 0, run.n_rows, int(k[0]), int(k[-1])))
        dvs[path] = sorted(rng.choice(run.n_rows, size=run.n_rows // (i + 2), replace=False).tolist()) if i != 1 else None
        filtered.append(_filter(run, dvs[path] or []))
    spec = DeduplicateMergeFunction.factory().create()
    factory = KeyValueFileReaderFactory(schema, dv_factory=lambda name: dvs[name])
    batches = []
    for section in IntervalPartition(metas).partition():
        rd = MergeTreeReaders.reader_for_section(section, factory, None, spec.with_read_fields(mask))
        try:
            while True:
                b = rd.read_batch()
                if b is None:
                    break
                batches.append(b)
        finally:
            rd.close()
    got = KeyValueBatch.from_rows(schema, [row for b in batches for row in b.to_rows()]).project(mask)
    want = pyoracle.merge(schema, spec, filtered).project(mask)
    assert got.equals(want), got.first_difference(want)
