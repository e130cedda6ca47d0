"""Handles keep what they use alive: a merge runs after its schema, spec and runs were freed, a rebind follows the free
of the previous runs, a view outlives the run it was sliced from, and a Parquet reader outlives its schema.  Every
result is compared bit for bit with the oracle (or with what was fetched before the free)."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import KeyValueBatch
from paimon_b200.compact_rewriter import KeyValueDataFileWriter
from paimon_b200.format import ParquetFileRecordReader, read_section
from paimon_b200.merge_function import DeduplicateMergeFunction, PartialUpdateMergeFunction
from paimon_b200.sort_merge_reader import (SortedRunReader, SortMergeReader, _SchemaHandle, apply_deletion_vector,
                                           export_arrow, fetch_run, slice_rows)
from paimon_b200.types import DataField, KeyValueSchema, RowType

from parquet_util import arrow_to_batch, write_kv_parquet

pytestmark = pytest.mark.gpu

VT = RowType((DataField("pk", "BIGINT", False), DataField("a", "BIGINT", True), DataField("b", "VARCHAR(24)", True),
              DataField("g", "INT", True), DataField("d", "DOUBLE", True), DataField("s", "VARCHAR(24)", True)))
SCHEMA = KeyValueSchema.of(VT, ["pk"])


def _spec(engine):
    if engine == "deduplicate":
        return DeduplicateMergeFunction.factory().create()
    return PartialUpdateMergeFunction.factory({"fields.g.sequence-group": "a,b"}, VT, ["pk"]).create()


def _runs(n_runs, total, seed, engine="deduplicate"):
    runs = datagen.make_runs(SCHEMA, n_runs, total, seed=seed, null_prob=0.3,
                             delete_prob=0.1 if engine == "deduplicate" else 0.0)
    g = SCHEMA.n_key + 2 + VT.field_names().index("g")
    for run in runs:                      # few group sequence values: ties and reversals between runs are common
        run.columns[g].data = (np.abs(run.columns[g].data) % 3).astype(run.columns[g].data.dtype)
    return runs


def _without(batch, deleted):
    gone = set(deleted)
    return KeyValueBatch.from_rows(batch.schema, [row for i, row in enumerate(batch.to_rows()) if i not in gone])


def _free(fn, handle):
    assert fn(handle) == 0, N.load().pg_last_error()


@pytest.mark.parametrize("engine", ["deduplicate", "partial-update"])
def test_merge_after_every_input_handle_is_freed(tmp_path, engine):
    lib = N.init(0)
    spec = _spec(engine)
    runs = _runs(5, 12000, seed=41, engine=engine)
    deleted = sorted(np.random.default_rng(3).choice(runs[4].n_rows, runs[4].n_rows // 4, replace=False).tolist())
    want = pyoracle.merge(SCHEMA, spec, runs[:4] + [_without(runs[4], deleted)], pyoracle.SORT_LOSER_TREE)

    path = str(tmp_path / "r3.parquet")
    write_kv_parquet(runs[3], path)
    section, _ = read_section(SCHEMA, [(open(path, "rb").read(), 0)], 1)
    dv_input = SortedRunReader(SCHEMA, runs[4])
    dv = apply_deletion_vector(SCHEMA, dv_input, deleted)
    dv_input.close()
    rd = SortMergeReader([SortedRunReader(SCHEMA, b) for b in runs[:3]] + section + [dv], spec)
    try:
        _free(lib.pg_schema_free, rd._schema_h.handle)
        rd._schema_h.handle = 0
        _free(lib.pg_merge_spec_free, rd._spec_h)
        rd._spec_h = 0
        for r in rd.readers:
            _free(lib.pg_run_free, r._handle)
            r._handle = 0
        rd.execute()
        got = rd.fetch()
        _free(lib.pg_merge_free, rd._merge_h)
        rd._merge_h = 0
    finally:
        rd.close()
    assert got.equals(want), got.first_difference(want)


def test_rebind_after_the_previous_runs_are_freed():
    lib = N.init(0)
    spec = _spec("deduplicate")
    set_a, set_b = _runs(3, 6000, seed=43), _runs(3, 6000, seed=44)
    starts = [3, 130, 1001]
    want = pyoracle.merge(SCHEMA, spec, [slice_rows(b, s, b.n_rows) for b, s in zip(set_b, starts)],
                          pyoracle.SORT_LOSER_TREE)
    rd = SortMergeReader([SortedRunReader(SCHEMA, b) for b in set_a], spec)
    try:
        rd.execute()
        for r in rd.readers:
            _free(lib.pg_run_free, r._handle)
            r._handle = 0
        # a rebind that fails leaves nothing bound
        with pytest.raises(N.PaimonGpuError, match="unknown run handle"):
            N.check(lib.pg_merge_rebind(rd._merge_h, (C.c_uint64 * 1)(12345), 1, None))
        rd.execute()
        assert rd.fetch().n_rows == 0
        rd.rebind([SortedRunReader(SCHEMA, b) for b in set_b], starts)
        rd.execute()
        got = rd.fetch()
        rd.execute()                                       # a re-execute takes the runs again while they are open
        again = rd.fetch()
        for r in rd.readers:
            r.close()
        with pytest.raises(N.PaimonGpuError, match="has been freed"):
            rd.execute()
    finally:
        rd.close()
    assert got.equals(want), got.first_difference(want)
    assert again.equals(want), again.first_difference(want)


def test_a_view_outlives_its_source_run(tmp_path):
    lib = N.init(0)
    runs = _runs(2, 8000, seed=45)
    sh = _SchemaHandle(SCHEMA, 0)
    src = SortedRunReader(SCHEMA, runs[0])
    view = C.c_uint64(0)
    try:
        full = fetch_run(SCHEMA, src._open(sh.handle))
        row_lo, row_hi = 201, full.n_rows - 17
        start = C.c_int64(0)
        N.check(lib.pg_run_slice(src._handle, row_lo, row_hi, C.byref(view), C.byref(start)))
        src.close()
        lo = row_lo - start.value
        want = slice_rows(full, lo, row_hi)

        got = fetch_run(SCHEMA, view.value)
        assert got.equals(want), got.first_difference(want)
        got = arrow_to_batch(SCHEMA, pa.Table.from_batches([export_arrow(SCHEMA, view.value)]))
        assert got.equals(want), got.first_difference(want)
        path = str(tmp_path / "view.parquet")
        KeyValueDataFileWriter(SCHEMA, path, level=0).write(view.value)
        got = arrow_to_batch(SCHEMA, pq.read_table(path))
        assert got.equals(want), got.first_difference(want)

        spec = _spec("deduplicate")
        merge_want = pyoracle.merge(SCHEMA, spec, [slice_rows(full, row_lo, row_hi), runs[1]], pyoracle.SORT_LOSER_TREE)
        view_reader = SortedRunReader.from_native_run(SCHEMA, row_hi - lo, view.value)
        rd = SortMergeReader([view_reader, SortedRunReader(SCHEMA, runs[1])], spec, start_rows=[start.value, 0])
        view.value = 0                                     # the merge reader frees the view with its runs
        try:
            rd.execute()
            got = rd.fetch()
        finally:
            rd.close()
        assert got.equals(merge_want), got.first_difference(merge_want)
    finally:
        if view.value:
            lib.pg_run_free(view.value)
        src.close()
        sh.close()


def test_a_parquet_reader_outlives_its_schema(tmp_path):
    lib = N.init(0)
    path = str(tmp_path / "f.parquet")
    write_kv_parquet(_runs(1, 5000, seed=46)[0], path)
    rd = ParquetFileRecordReader(SCHEMA, open(path, "rb").read())
    try:
        _free(lib.pg_schema_free, rd._schema_h.handle)
        rd._schema_h.handle = 0
        got = rd.read_batch()
    finally:
        rd.close()
    want = arrow_to_batch(SCHEMA, pq.read_table(path))
    assert got.equals(want), got.first_difference(want)
