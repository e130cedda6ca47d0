"""Runs opened from device memory (PG_MEM_DEVICE) through every entry point that takes a run, in the layouts of
tests/device_runs.py, and the bench's own device-generated inputs.

Every case compares with the oracle or a numpy model of the host mirror (the tensors read back with .cpu()), and where
a host-opened run of the same bytes exists, the device-opened run must give byte-identical results: values (NULL slots
included), offsets, and validity bits below n_rows.  Needs an H100."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest
import torch

import device_runs as D
import file_index_reference as R
import stats_reference as S
from bench_shapes import PARQUET_GROUP_ROWS, PARQUET_PAGE_ROWS, schema_c4
from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import Column, KeyValueBatch, pack_validity, unpack_validity
from paimon_b200.compact_rewriter import file_column_names
from paimon_b200.merge_function import (AggregateMergeFunction, DeduplicateMergeFunction, FirstRowMergeFunction,
                                        PartialUpdateMergeFunction)
from paimon_b200.sort_merge_reader import (SortedRunReader, SortMergeReader, _SchemaHandle, export_arrow, fetch_run,
                                           slice_rows)
from paimon_b200.types import DataField, KeyValueSchema, PhysicalType, RowType, is_varlen

from parquet_util import arrow_to_batch
from test_gpu_orc_write import check_file as orc_check_file
from test_gpu_parquet_write_stats import _device_encode, _raw_of_model, footer_of

pytestmark = pytest.mark.gpu
P = PhysicalType
PG_ERR_INVALID = 1
SIZES = [0, 1, 7, 8, 10_000]


@pytest.fixture(scope="module")
def lib():
    return N.init(0)


def names_array(schema):
    names = file_column_names(schema)
    return (C.c_char_p * len(names))(*[x.encode() for x in names])


def identical(a, b):
    """Byte identity of two fetched batches: values under NULL slots too, offsets, payload, validity below n_rows."""
    assert a.n_rows == b.n_rows
    n = a.n_rows
    for ci, (x, y) in enumerate(zip(a.columns, b.columns)):
        assert n == 0 or (x.valid is None) == (y.valid is None), ci
        if x.valid is not None and y.valid is not None:
            assert np.array_equal(unpack_validity(x.valid, n), unpack_validity(y.valid, n)), ci
        if x.offsets is not None:
            ox, oy = np.asarray(x.offsets[: n + 1]), np.asarray(y.offsets[: n + 1])
            assert np.array_equal(ox - ox[0], oy - oy[0]), ci
            assert x.data[ox[0]:ox[-1]].tobytes() == y.data[oy[0]:oy[-1]].tobytes(), ci
        else:
            assert x.data[:n].tobytes() == y.data[:n].tobytes(), ci


def open_both(sh, run, layout, big_base=False):
    """(device run, its host mirror, device handle, handle of the mirror opened from host memory)"""
    dr = D.DeviceRun(run, layout, big_base)
    mirror = dr.mirror()
    dev, host = dr.reader(), SortedRunReader(run.schema, mirror)
    return dr, mirror, dev, host, dev._open(sh.handle), host._open(sh.handle)


# ---------------------------------------------------------------------------------------------- open / layout / fetch

@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("layout", D.LAYOUTS)
def test_open_layout_fetch(lib, layout, n):
    run = D.model_runs(1, n, seed=n + 3)[0]
    schema = run.schema
    sh = _SchemaHandle(schema, 0)
    dr, mirror, dev, host, hd, hh = open_both(sh, run, layout, big_base=n == 10_000)
    try:
        rows = C.c_int64(0)
        db = np.zeros(schema.n_cols, np.int64)
        N.check(lib.pg_run_layout(hd, C.byref(rows), db.ctypes.data, None, schema.n_cols))
        assert rows.value == n
        for c, col in enumerate(mirror.columns):
            if col.offsets is not None:
                assert db[c] == (int(col.offsets[n]) - int(col.offsets[0]) if n else 0), (c, db[c])
        got = fetch_run(schema, hd)
        assert got.equals(mirror), got.first_difference(mirror)
        assert got.equals(run), got.first_difference(run)
        identical(got, fetch_run(schema, hh))
    finally:
        dev.close(); host.close(); sh.close()


def test_open_refusals(lib):
    run = D.model_runs(1, 100, seed=4)[0]
    schema = run.schema
    sh = _SchemaHandle(schema, 0)
    s_col = schema.n_key + 2 + schema.value_type.index_of("s")
    try:
        def status(cols, mem=N.PG_MEM_DEVICE):
            pc = (N.PgColumn * schema.n_cols)(*[N.PgColumn(c.data or None, c.offsets or None, c.validity or None)
                                                for c in cols])
            h = C.c_uint64(0)
            st = lib.pg_run_open(sh.handle, C.byref(N.PgRunDesc(run.n_rows, pc)), mem, C.byref(h))
            if st == 0:
                lib.pg_run_free(h.value)
            return st
        dr = D.DeviceRun(run, "based")
        assert status(dr.columns) == 0
        for kind in ("data", "offsets", "validity"):
            cols = [D.DeviceColumn(c.data, c.offsets, c.validity) for c in dr.columns]
            setattr(cols[s_col], kind, getattr(cols[s_col], kind) + 8)
            assert status(cols) == PG_ERR_INVALID, kind
        cols = [D.DeviceColumn(c.data, c.offsets, c.validity) for c in dr.columns]
        cols[s_col].offsets = 0
        assert status(cols) == PG_ERR_INVALID
        # offsets[n] below offsets[0] (s is the first var-len column of a based run: its offsets start at 13)
        t, off, _ = dr._spans[s_col][1]
        view = t[off:off + 4 * (run.n_rows + 1)].view(torch.int32)
        assert int(view[0]) == 13
        view[run.n_rows] = 5
        assert status(dr.columns) == PG_ERR_INVALID
        # the host path refuses the same offsets
        host = dr.mirror()
        keep = [np.ascontiguousarray(c.data) for c in host.columns]
        pc = (N.PgColumn * schema.n_cols)(*[N.PgColumn(k.ctypes.data, None if c.offsets is None else
                                                       np.ascontiguousarray(c.offsets).ctypes.data,
                                                       None if c.valid is None else c.valid.ctypes.data)
                                            for k, c in zip(keep, host.columns)])
        h = C.c_uint64(0)
        assert lib.pg_run_open(sh.handle, C.byref(N.PgRunDesc(run.n_rows, pc)), N.PG_MEM_HOST, C.byref(h)) == PG_ERR_INVALID
    finally:
        sh.close()


# ---------------------------------------------------------------------------------------------- merge

def specs():
    vt = D.schema_all().value_type
    return {
        "dedup": DeduplicateMergeFunction.factory().create(),
        "first_row": FirstRowMergeFunction.factory().create(),
        "pu_seq_group": PartialUpdateMergeFunction.factory({"fields.g.sequence-group": "v,s"}, vt, ["k"]).create(),
        "agg_sum_max": AggregateMergeFunction.factory({"fields.d.aggregate-function": "sum",
                                                       "fields.v.aggregate-function": "max"}, vt, ["k"]).create(),
        "drop_delete": DeduplicateMergeFunction.factory().create().with_drop_delete(),
    }


MERGE_CASES = [(1, 0, "separate"), (1, 1, "based"), (2, 7, "arena"), (2, 8, "dirty"), (8, 1, "aliased"),
               (32, 8, "based")] + [(8, 10_000, lay) for lay in D.LAYOUTS] + [(32, 1000, "dirty")]


def merge_batch(schema, spec, readers, start_rows=None):
    rd = SortMergeReader(readers, spec, start_rows=start_rows)
    try:
        rd.execute()
        return rd.fetch()
    finally:
        rd.close()


@pytest.mark.parametrize("k,n,layout", MERGE_CASES)
@pytest.mark.parametrize("engine", sorted(specs()))
def test_merge(engine, k, n, layout):
    """k runs, every third one opened from host memory, against the oracle; the same merge of the mirrors opened
    from host memory gives the same bytes."""
    spec = specs()[engine]
    runs = D.model_runs(k, n, seed=k * 31 + n, delete_prob=0.2 if engine in ("dedup", "drop_delete") else 0.0)
    schema = runs[0].schema
    dev = [D.DeviceRun(r, layout, big_base=(k, n) == (8, 10_000)) for r in runs]
    mirrors = [d.mirror() for d in dev]
    readers = [SortedRunReader(schema, m) if r % 3 == 1 else d.reader() for r, (d, m) in enumerate(zip(dev, mirrors))]
    got = merge_batch(schema, spec, readers)
    want = pyoracle.merge(schema, spec, [D.clean(m) for m in mirrors], pyoracle.SORT_LOSER_TREE)
    assert got.equals(want), got.first_difference(want)
    identical(got, merge_batch(schema, spec, [SortedRunReader(schema, m) for m in mirrors]))


@pytest.mark.parametrize("layout", ["based", "arena"])
def test_slices_and_rebind(layout):
    """pg_run_slice views of device runs with row bounds off the 128-row grid, merged through pg_merge_rebind with
    the views' start rows."""
    lib = N.init(0)
    runs = D.model_runs(6, 9000, seed=17)
    schema = runs[0].schema
    spec = DeduplicateMergeFunction.factory().create()
    dev = [D.DeviceRun(r, layout, big_base=True) for r in runs]
    mirrors = [d.mirror() for d in dev]
    bounds = [(0, 9000), (1, 8999), (127, 4097), (129, 130), (333, 333), (5000, 8191)]
    rd = SortMergeReader([dev[0].reader()], spec)
    base = rd.readers
    try:
        handles = [d.reader()._open(rd._schema_h.handle) for d in dev]
        views, starts = [], []
        for h, (lo, hi) in zip(handles, bounds):
            v, s = C.c_uint64(0), C.c_int64(0)
            N.check(lib.pg_run_slice(h, lo, hi, C.byref(v), C.byref(s)))
            assert s.value == lo % 128
            views.append(SortedRunReader.from_native_run(schema, hi - (lo & ~127), v.value))
            starts.append(s.value)
        for h in handles:
            lib.pg_run_free(h)                                 # the views keep their sources alive
        rd.rebind(views, starts)
        for r in base:
            r.close()
        rd.execute()
        got = rd.fetch()
        for v, (lo, hi), m in zip(views, bounds, mirrors):
            part = fetch_run(schema, v._handle)
            assert part.equals(slice_rows(m, lo & ~127, hi))
    finally:
        rd.close()
    want = pyoracle.merge(schema, spec, [slice_rows(D.clean(m), lo, hi) for m, (lo, hi) in zip(mirrors, bounds)],
                          pyoracle.SORT_LOSER_TREE)
    assert got.equals(want), got.first_difference(want)


# ---------------------------------------------------------------------------------------------- deletion vectors

DV_SCHEMA = KeyValueSchema.of(RowType((DataField("k", "BIGINT", False), DataField("d", "DOUBLE", True),
                                       DataField("s", "STRING", True))), ["k"])


def dv_run(n, seed):
    rng = np.random.default_rng(seed)
    k = Column(P.INT64, np.arange(n, dtype=np.int64) * 3)
    d_valid, s_valid = rng.random(n) >= 0.3, rng.random(n) >= 0.3
    lens = rng.integers(0, 9, n) * s_valid
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    s = Column(P.STRING, rng.integers(0x21, 0x7f, int(offs[-1]), dtype=np.uint8), offs.astype(np.int32),
               pack_validity(s_valid))
    return KeyValueBatch(DV_SCHEMA, [k, Column(P.INT64, np.arange(n, dtype=np.int64)), Column(P.INT8, np.zeros(n, np.int8)),
                                     k, Column(P.DOUBLE, rng.uniform(-9, 9, n), None, pack_validity(d_valid)), s])


def take_rows(batch, rows):
    """Rows `rows` (ascending) of a clean host batch, vectorised."""
    cols = []
    for c in batch.columns:
        valid = None if c.valid is None else pack_validity(unpack_validity(c.valid, len(c))[rows])
        if c.offsets is None:
            cols.append(Column(c.type, np.asarray(c.data)[rows], None, valid))
            continue
        o = np.asarray(c.offsets, np.int64)
        lens = (o[1:] - o[:-1])[rows]
        new = np.zeros(len(rows) + 1, np.int64)
        np.cumsum(lens, out=new[1:])
        idx = np.repeat(o[:-1][rows] - new[:-1], lens) + np.arange(int(new[-1]))
        cols.append(Column(c.type, np.asarray(c.data)[idx], new.astype(np.int32), valid))
    return KeyValueBatch(batch.schema, cols)


def deleted_flags(pattern, n_bits, rng):
    if pattern == "none":
        return np.zeros(n_bits, bool)
    if pattern == "all":
        return np.ones(n_bits, bool)
    if pattern == "alternating":
        return np.arange(n_bits) % 2 == 1
    return rng.random(n_bits) < 0.4


def check_dv(lib, sh, h, mirror, n, n_bits, pattern, rng):
    flags = deleted_flags(pattern, n_bits, rng)
    bitmap = np.packbits(flags, bitorder="little") if n_bits else np.zeros(1, np.uint8)
    bitmap = np.concatenate([bitmap, np.zeros(8, np.uint8)])
    out = C.c_uint64(0)
    N.check(lib.pg_run_apply_deletion_vector(h, bitmap.ctypes.data, n_bits, C.byref(out)))
    try:
        got = fetch_run(DV_SCHEMA, out.value)
    finally:
        lib.pg_run_free(out.value)
    keep = np.ones(n, bool)
    keep[: min(n, n_bits)] = ~flags[:n]
    want = take_rows(D.clean(mirror), np.flatnonzero(keep))
    assert got.equals(want), (n_bits, pattern, got.first_difference(want))
    m = got.n_rows
    for c in got.columns:                                # no validity bit past the output's last row
        if c.valid is not None and m % 8:
            assert np.unpackbits(c.valid[m // 8: m // 8 + 1], bitorder="little")[m % 8:].sum() == 0


@pytest.mark.parametrize("n", [0, 1, 8, 4095, 4096, 4097, 4 * (1 << 20) + 1])
@pytest.mark.parametrize("layout", D.LAYOUTS)
def test_deletion_vector(lib, layout, n):
    """Past 4 Mi rows each thread of k_scan_block_prefix sums more than one block."""
    rng = np.random.default_rng(n)
    dr = D.DeviceRun(dv_run(n, n + 1), layout, big_base=n > 4096)
    mirror = dr.mirror()
    sh = _SchemaHandle(DV_SCHEMA, 0)
    rd = dr.reader()
    try:
        h = rd._open(sh.handle)
        if n <= 4097:
            cases = [(b, p) for b in sorted({0, max(n - 3, 0), n, n + 13}) for p in ("none", "all", "alternating", "random")]
        else:
            cases = [(n, "random"), (n - 3, "alternating"), (n + 13, "all"), (0, "none")]
        for n_bits, pattern in cases:
            check_dv(lib, sh, h, mirror, n, n_bits, pattern, rng)
    finally:
        rd.close(); sh.close()


def test_deletion_vector_20M_rows(lib):
    n = 20_000_000
    rng = np.random.default_rng(20)
    dr = D.DeviceRun(dv_run(n, 21), "based", big_base=True)
    mirror = dr.mirror()
    sh = _SchemaHandle(DV_SCHEMA, 0)
    rd = dr.reader()
    try:
        h = rd._open(sh.handle)
        check_dv(lib, sh, h, mirror, n, n + 13, "random", rng)
    finally:
        rd.close(); sh.close()


# ---------------------------------------------------------------------------------------------- encoders

ENC_CASES = [(lay, row0, cnt) for lay in ("dirty", "based", "arena") for row0, cnt in ((0, -1), (8, 3001), (1000, 0))]


@pytest.mark.parametrize("layout,row0,cnt", ENC_CASES)
def test_parquet_encode(lib, layout, row0, cnt):
    """pg_parquet_encode, none and zstd-1: pyarrow reads the model's rows back; footer and file statistics follow
    stats_reference (NULL slots never reach min / max, tail validity bits never reach null counts)."""
    run = D.model_runs(1, 5000, seed=41)[0]
    schema = run.schema
    dr = D.DeviceRun(run, layout, big_base=True)
    model = D.clean(dr.mirror())
    n = model.n_rows - row0 if cnt < 0 else cnt
    writer = dict(page_rows=64, row_group_rows=1000)
    sh = _SchemaHandle(schema, 0)
    rd = dr.reader()
    try:
        h = rd._open(sh.handle)
        opts = N.PgParquetWriteOptions(writer["row_group_rows"], writer["page_rows"])
        for codec in (None, 6):
            blob, meta, cols = _device_encode(lib, h, schema.n_cols, names_array(schema), row0, n, codec, opts)
            assert meta.n_rows == n
            back = arrow_to_batch(schema, pq.read_table(pa.BufferReader(blob)))
            want = slice_rows(model, row0, row0 + n)
            assert back.equals(want), back.first_difference(want)
            assert footer_of(blob, schema.physical_types()) == S.footer_stats(model, row0, n, **writer)
            for c, (t, st) in enumerate(zip(schema.physical_types(), S.file_stats(model, row0, n))):
                raw = _raw_of_model(t, st)
                assert cols[c][:2] == raw[:2] and (not raw[1] or cols[c][2:] == raw[2:]), (codec, c, cols[c], raw)
    finally:
        rd.close(); sh.close()


@pytest.mark.parametrize("layout,row0,cnt", ENC_CASES)
def test_orc_encode(tmp_path, layout, row0, cnt):
    run = D.model_runs(1, 5000, seed=43)[0]
    schema = run.schema
    dr = D.DeviceRun(run, layout, big_base=True)
    model = D.clean(dr.mirror())
    n = model.n_rows - row0 if cnt < 0 else cnt
    path = str(tmp_path / "f.orc")
    N.init(0)
    sh = _SchemaHandle(schema, 0)
    rd = dr.reader()
    try:
        from paimon_b200.compact_rewriter import KeyValueDataFileWriter
        written = KeyValueDataFileWriter(schema, path, level=0, file_format="orc", stripe_rows=1000).write(
            rd._open(sh.handle), row0, n)
    finally:
        rd.close(); sh.close()
    orc_check_file(schema, slice_rows(model, row0, row0 + n), path, written, 1000)


BLOOM = [("v", "BIGINT"), ("d", "DOUBLE"), ("s", "STRING"), ("i", "INT"), ("y", "BINARY")]


@pytest.mark.parametrize("layout", ["dirty", "based", "arena"])
def test_bloom_filter(lib, layout):
    """pg_bloom_filter_build skips NULL slots, whatever they hold, and takes the payload at the run's offsets."""
    run = D.model_runs(1, 3000, seed=47)[0]
    schema = run.schema
    dr = D.DeviceRun(run, layout, big_base=True)
    model = D.clean(dr.mirror())
    sh = _SchemaHandle(schema, 0)
    rd = dr.reader()
    try:
        h = rd._open(sh.handle)
        for name, logical in BLOOM:
            c = schema.n_key + 2 + schema.value_type.index_of(name)
            for row0, cnt in ((0, -1), (16, 1001)):
                end = model.n_rows if cnt < 0 else row0 + cnt
                vals = model.columns[c].to_pylist()[row0:end]
                if logical == "DOUBLE":
                    vals = [None if v is None else ("bits", int(np.float64(v).view(np.uint64))) for v in vals]
                want = R.filter_of(logical, vals, items=500)
                buf = np.zeros(len(want), np.uint8)
                spec = N.PgBloomFilterSpec(c, 500, 0.1)
                N.check(lib.pg_bloom_filter_build(h, row0, cnt, 1, C.byref(spec), (C.c_void_p * 1)(buf.ctypes.data),
                                                  (C.c_int64 * 1)(len(want))))
                assert buf.tobytes() == want, (name, row0)
    finally:
        rd.close(); sh.close()


# ---------------------------------------------------------------------------------------------- Arrow export

def check_export(schema, handle, model, row0, cnt):
    rb = export_arrow(schema, handle, row0, cnt)
    assert rb.num_rows == cnt
    for f, arr, col in zip(schema.file_fields(), rb.columns, model.columns):
        pt = P(col.type)
        if pt == P.BOOL:
            assert arr.type == pa.bool_()
        if pt == P.BINARY:
            assert arr.type == pa.binary()
        if is_varlen(pt):
            assert np.frombuffer(arr.buffers()[1], np.int32)[0] == 0
        assert rb.schema.field(f.name).nullable == (f.nullable or col.valid is not None)
    got = arrow_to_batch(schema, pa.Table.from_batches([rb], schema=rb.schema))
    want = slice_rows(model, row0, row0 + cnt)
    assert got.equals(want), (row0, cnt, got.first_difference(want))


@pytest.mark.parametrize("layout", D.LAYOUTS)
def test_arrow_export(lib, layout):
    run = D.model_runs(1, 3000, seed=53)[0]
    schema = run.schema
    dr = D.DeviceRun(run, layout, big_base=True)
    model = D.clean(dr.mirror())
    sh = _SchemaHandle(schema, 0)
    rd = dr.reader()
    try:
        h = rd._open(sh.handle)
        for row0, cnt in ((0, 3000), (3, 1), (13, 2500), (999, 0), (3000, 0), (2997, 3)):
            check_export(schema, h, model, row0, cnt)
        v, s = C.c_uint64(0), C.c_int64(0)
        N.check(lib.pg_run_slice(h, 301, 2711, C.byref(v), C.byref(s)))
        try:
            view = slice_rows(model, 301 - s.value, 2711)
            for row0, cnt in ((0, view.n_rows), (s.value, 2711 - 301), (s.value + 5, 77), (9, 0)):
                check_export(schema, v.value, view, row0, cnt)
        finally:
            lib.pg_run_free(v.value)
    finally:
        rd.close(); sh.close()


# ---------------------------------------------------------------------------------------------- the bench's inputs

def bench_spec(name, schema):
    if name == "c3agg":
        opts = {f"fields.{f.name}.aggregate-function": "sum" for f in schema.value_type.fields
                if f.name != "pk" and f.physical.name in ("INT64", "DOUBLE")}
        return AggregateMergeFunction.factory(opts, schema.value_type, ["pk"]).create()
    if name.startswith("c3"):
        return PartialUpdateMergeFunction.factory({}, schema.value_type, ["pk"]).create()
    spec = DeduplicateMergeFunction.factory().create()
    return spec.with_drop_delete() if name == "c4" else spec


BENCH = {  # name: (schema, runs, rows per run, null_prob, delete_prob)
    "c2": (datagen.schema_c2, 8, 2_000_000, 0.0, 0.0),
    "c3": (datagen.schema_c3, 16, 200_000, 0.5, 0.0),
    "c3agg": (datagen.schema_c3, 16, 200_000, 0.5, 0.0),
    "c4": (schema_c4, 32, 100_000, 0.5, 0.05),
}


def bench_runs(name, seed=0):
    make, k, per_run, null_prob, delete_prob = BENCH[name]
    schema = make()
    dev = torch.device("cuda", 0)
    key_space = max(k * per_run // 2, per_run)
    out = []
    for r in range(k):
        cols, keep, _, _, _ = D.gen_device_run(schema, r, per_run, key_space, null_prob, seed, dev, delete_prob)
        out.append((SortedRunReader.from_device(schema, per_run, cols, keepalive=keep),
                    D.bench_mirror(schema, per_run, cols, keep)))
    torch.cuda.synchronize()
    return schema, out


@pytest.mark.parametrize("name", sorted(BENCH))
def test_bench_merge(name):
    N.init(0)
    schema, runs = bench_runs(name)
    spec = bench_spec(name, schema)
    got = merge_batch(schema, spec, [r for r, _ in runs])
    want = pyoracle.merge(schema, spec, [D.clean(m) for _, m in runs], pyoracle.SORT_LOSER_TREE)
    assert got.equals(want), got.first_difference(want)


def test_bench_parquet_encode(lib):
    """One C3 run at the bench's page and row-group limits, read back by pyarrow."""
    schema, runs = bench_runs("c3")
    rd, mirror = runs[0]
    for r, _ in runs[1:]:
        r.close()
    sh = _SchemaHandle(schema, 0)
    try:
        opts = N.PgParquetWriteOptions(PARQUET_GROUP_ROWS, PARQUET_PAGE_ROWS)
        blob, meta, _ = _device_encode(lib, rd._open(sh.handle), schema.n_cols, names_array(schema), 0, -1, None, opts)
    finally:
        rd.close(); sh.close()
    back = arrow_to_batch(schema, pq.read_table(pa.BufferReader(blob)))
    model = D.clean(mirror)
    assert back.equals(model), back.first_difference(model)
    assert footer_of(blob, schema.physical_types()) == S.footer_stats(model, 0, model.n_rows, PARQUET_PAGE_ROWS,
                                                                      PARQUET_GROUP_ROWS)
