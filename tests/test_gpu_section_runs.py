"""The decoded runs of a section: the Parquet and the ORC decoder lay out the same runs from the same rows (read columns,
NULL rows of a field some files lack, absent unread columns, `decoded_bytes`), and a deletion vector applied to a
projected run keeps the projection."""
import ctypes as C

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
from paimon_b200.sort_merge_reader import apply_deletion_vector
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
