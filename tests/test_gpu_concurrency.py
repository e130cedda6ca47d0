"""The library under concurrent callers and recycled device buffers.  Needs an H100.

include/paimon_gpu.h promises that the library is re-entrant across handles and that a handle may be freed while
another thread is inside a call on it; the JNI layer, RangeStreamingMergeReader and the end-to-end leg of bench.py rely
on it.  Here 8 threads run whole pipelines at once (decode from host and from device bytes, deletion vector, merge,
rebind, slices, Arrow export, Parquet and ORC encode, bloom-filter file index), handles cross threads that never called
pg_init, and handles are freed under calls on them.  Every result is checked against the plain references the other
tests use (pyoracle.merge, pyarrow, the bloom-filter model), and everything computed under concurrency must be
bit-identical to the same pipeline run on one thread: the encoders are deterministic, so every file is compared byte for
byte.

Before each round the recycled-buffer cache is filled with buffers of 0xA5 bytes (dirty_cache), so that every device
buffer the calls take is dirty: a kernel that relies on zeroed memory fails here rather than only after some earlier
test happened to leave the wrong garbage behind.  test_dirty_cache_single_thread runs each device path once that way."""
import ctypes as C
import io
import os
import threading

import numpy as np
import pyarrow as pa
import pyarrow.orc as porc
import pyarrow.parquet as pq
import pytest

import file_index_reference as R
from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import Column, KeyValueBatch, pack_validity, unpack_validity
from paimon_b200.compact_rewriter import KeyValueDataFileWriter, file_column_names
from paimon_b200.file_index import DataFileIndexWriter, FileIndexOptions
from paimon_b200.format import FileUpload, read_section
from paimon_b200.merge_function import (AggregateMergeFunction, DeduplicateMergeFunction, FirstRowMergeFunction,
                                        PartialUpdateMergeFunction)
from paimon_b200.merge_tree_readers import concat_batches
from paimon_b200.sort_merge_reader import (RangeStreamingMergeReader, SortedRunReader, SortMergeReader, _SchemaHandle,
                                           apply_deletion_vector, export_arrow, fetch_run, fetch_slice, merge_runs,
                                           slice_rows)
from paimon_b200.types import DataField, KeyValueSchema, RowType

from parquet_util import arrow_to_batch, to_arrow, write_kv_parquet

pytestmark = pytest.mark.gpu

WORKERS, ROUNDS = 8, 2
DIRTY = 0xA5
LARGEST = 48 << 20             # above the largest device buffer any call below takes (a run of ~20k wide rows)


# ------------------------------------------------------------------------------------------------ the dirty cache

def dirty_cache(copies: int = WORKERS, largest: int = LARGEST):
    """Fill the recycled-buffer cache with buffers of 0xA5 bytes, `copies` of each size.

    Runs, uploads and the temporaries of every decode, deletion vector and encode come from that cache, and buf_take
    (api.cu) serves a request of b bytes with any cached buffer of b to 1.5 b + 1 MiB bytes, as it is.  The cache is
    emptied first (pg_trim), then uploads of 0xA5 bytes (pg_files_upload_begin, wait, free) leave buffers of the sizes
    s_0 = 256, s_i+1 = ceil(1.4 s_i), up to the first one at or above `largest`, in it (an upload of n bytes takes
    n + 64).  A request of b bytes in (s_i-1, s_i] finds s_i's buffer, since s_i <= 1.4 s_i-1 < 1.4 b < 1.5 b, and one
    of at most 256 bytes finds s_0's: every request up to `largest` is served dirty, by one of `copies` buffers of its
    size, as long as no more than `copies` requests of one size are in flight.  The sizes sum to less than
    3.5 x 1.4 x largest, 8 x 235 MiB in all for the defaults: far below the cache's default limit of 16 GiB."""
    lib = N.init(0)
    N.check(lib.pg_trim())
    sizes, s = [], 256
    while True:
        sizes.append(s)
        if s >= largest:
            break
        s = -(-s * 14 // 10)
    src = np.full(sizes[-1], DIRTY, np.uint8)
    up = FileUpload([(src[: n - 64], 0) for n in sizes for _ in range(copies)])
    up.wait()
    up.close()
    assert copies * sum(sizes) < 2 << 30


# ------------------------------------------------------------------------------------------------ shapes and files

def decimal_schema_runs(schema, runs, names, modulo=10 ** 12):
    """DECIMAL(18, 4) values of datagen's runs brought inside the precision (their unscaled BIGINTs are any int64)."""
    out = []
    for b in runs:
        cols = list(b.columns)
        for ci, f in enumerate(schema.file_fields()):
            if f.name in names:
                cols[ci] = Column(cols[ci].type, (cols[ci].data % modulo) - modulo // 2, None, cols[ci].valid)
        out.append(KeyValueBatch(schema, cols))
    return out


def c3_schema():
    return datagen.schema_c3(n_i64=4, n_f64=3, n_str=4)


def all_types_schema():
    vt = RowType((DataField("pk", "BIGINT", False), DataField("l", "BIGINT", True), DataField("i", "INT", True),
                  DataField("dt", "DATE", True), DataField("dec", "DECIMAL(18,4)", True), DataField("d", "DOUBLE", True),
                  DataField("s", "STRING", True), DataField("bin", "BYTES", True)))
    return KeyValueSchema.of(vt, ["pk"])


def composite_schema():
    vt = RowType((DataField("a", "VARCHAR(20)", False), DataField("b", "BIGINT", False), DataField("v", "BIGINT", True),
                  DataField("s", "STRING", True), DataField("d", "DOUBLE", True)))
    return KeyValueSchema.of(vt, ["a", "b"])


def agg_schema():
    vt = RowType((DataField("pk", "BIGINT", False), DataField("dec", "DECIMAL(18,4)", True), DataField("i", "INT", True),
                  DataField("d", "DOUBLE", True), DataField("s", "STRING", True)))
    return KeyValueSchema.of(vt, ["pk"])


AGG_OPTIONS = {"fields.dec.aggregate-function": "sum", "fields.i.aggregate-function": "max",
               "fields.d.aggregate-function": "min", "fields.s.aggregate-function": "last_non_null_value"}

# kind -> (schema, spec, value-field names with a bloom filter, DECIMAL names, delete probability)
KINDS = {
    "c3_partial_update": (c3_schema, lambda s: PartialUpdateMergeFunction.factory({}, s.value_type, ["pk"]).create(),
                          ["i0", "s1"], (), 0.0),
    "all_types_dedup": (all_types_schema, lambda s: DeduplicateMergeFunction.factory().create(), ["l", "dt", "s", "bin"],
                        ("dec",), 0.1),
    "composite_key_dedup": (composite_schema, lambda s: DeduplicateMergeFunction.factory().create(), ["v", "s"], (), 0.15),
    "decimal_sum": (agg_schema, lambda s: AggregateMergeFunction.factory(AGG_OPTIONS, s.value_type, ["pk"]).create(),
                    ["i", "s"], ("dec",), 0.0),
}
KIND_NAMES = list(KINDS)

# how the pyarrow files of a section are written, file by file: codecs, dictionary and PLAIN strings,
# DELTA_BINARY_PACKED integers, data page V2
PARQUET_OPTS = [dict(compression="snappy"),
                dict(compression="zstd", use_dictionary=False, data_page_version="2.0"),
                dict(compression="gzip", data_page_size=4096),
                dict(compression="snappy", use_dictionary=False, data_page_version="2.0"),
                dict(compression="none", use_dictionary=False, column_encoding="delta"),
                dict(compression="zstd", row_group_size=1000, data_page_size=2048)]


def parquet_bytes(batch, opts):
    opts = dict(opts)
    if opts.get("column_encoding") == "delta":
        opts["column_encoding"] = {f.name: "DELTA_BINARY_PACKED" if f.physical.name in ("INT32", "INT64") else "PLAIN"
                                   for f in batch.schema.file_fields()}
    buf = io.BytesIO()
    write_kv_parquet(batch, buf, **opts)
    return buf.getvalue()


def orc_bytes(batch, codec):
    t = to_arrow(batch)
    if "dt" in t.column_names:
        t = t.set_column(t.column_names.index("dt"), "dt", t.column("dt").cast(pa.date32()))
    buf = io.BytesIO()
    porc.write_table(t, buf, compression=codec, stripe_size=64 * 1024, compression_block_size=65536)
    return buf.getvalue()


def device_bytes(schema, batch, fmt, tmp):
    """A data file written by the device encoder from a run of `batch`."""
    h = _SchemaHandle(schema, 0)
    rd = SortedRunReader(schema, batch)
    path = os.path.join(tmp, f"dev-{id(batch)}.{fmt}")
    try:
        kw = dict(page_rows=1500) if fmt == "parquet" else dict(file_format="orc", compression="zstd", stripe_rows=2500)
        KeyValueDataFileWriter(schema, path, level=0, **kw).write(rd._open(h.handle))
    finally:
        rd.close()
        h.close()
    return open(path, "rb").read()


class Case:
    """One worker's inputs: section A (pyarrow Parquet files) and section B (files of the device encoder, or ORC), three
    sorted runs of two files each; a deletion vector on run 0 of section A; and every reference the pipeline is checked
    against.  Variant 0 writes section B with the device's Parquet encoder, variant 1 as ORC (the device's ORC encoder
    for DECIMAL columns, pyarrow's otherwise)."""

    def __init__(self, kind, seed, variant, tmp):
        make_schema, make_spec, self.bloom, decimals, delete_prob = KINDS[kind]
        self.kind, self.seed = kind, seed
        self.schema = schema = make_schema()
        self.spec = make_spec(schema)
        self.sections, self.formats, self.runs = [], [], []
        for sec in range(2):
            files, runs = [], []
            for r in range(3):
                parts = []
                for f in range(2):
                    keys = np.arange(f * 12_000 + r + sec, f * 12_000 + 7_000 + 97 * r, 3, dtype=np.int64)
                    part = datagen.make_run(schema, 10 * r + f + 100 * sec, keys, seed=seed, null_prob=0.3,
                                            delete_prob=delete_prob)
                    part = decimal_schema_runs(schema, [part], decimals)[0]
                    if sec == 0:
                        data = parquet_bytes(part, PARQUET_OPTS[(seed + 2 * r + f) % len(PARQUET_OPTS)])
                    elif variant == 0:
                        data = device_bytes(schema, part, "parquet", tmp)
                    elif decimals:
                        data = device_bytes(schema, part, "orc", tmp)
                    else:
                        data = orc_bytes(part, ["zstd", "zlib", "lz4", "uncompressed"][(r + f) % 4])
                    files.append((data, r))
                    parts.append(part)
                runs.append(concat_batches(schema, parts))
            self.sections.append(files)
            self.formats.append("parquet" if sec == 0 or variant == 0 else "orc")
            self.runs.append(runs)
        rng = np.random.default_rng(seed)
        n0 = self.runs[0][0].n_rows
        self.deleted = np.sort(rng.choice(n0, n0 // 5, replace=False))
        keep = np.ones(n0, bool)
        keep[self.deleted] = False
        self.after_dv = take_rows(self.runs[0][0], keep)
        self.want = [pyoracle.merge(schema, self.spec, [self.after_dv] + self.runs[0][1:]),
                     pyoracle.merge(schema, self.spec, self.runs[1])]
        n = self.want[1].n_rows
        self.slices = [(1, 130), (127, 129 + 77), (n // 3 + 5, n - 9), (n - 3, n)]
        self.exports = [(3, 250), (129, n // 2), (n - 7, 7)]
        self.encoded = (8, n - 13)          # rows [row0, row0 + n_rows) of the merged batch that are written (row0: a multiple of 8)


def take_rows(batch, keep):
    cols = []
    for col in batch.columns:
        valid = None if col.valid is None else pack_validity(unpack_validity(col.valid, len(col))[keep])
        if col.offsets is not None:
            o = np.asarray(col.offsets, np.int64)
            lens = np.diff(o)[keep]
            data = np.concatenate([col.data[o[i]:o[i + 1]] for i in np.flatnonzero(keep)]) if keep.any() else \
                np.zeros(0, np.uint8)
            offs = np.zeros(len(lens) + 1, np.int64)
            np.cumsum(lens, out=offs[1:])
            cols.append(Column(col.type, data, offs.astype(np.int32), valid))
        else:
            cols.append(Column(col.type, np.asarray(col.data)[: len(keep)][keep], None, valid))
    return KeyValueBatch(batch.schema, cols)


def normalise(table):
    """A table read back by pyarrow with DECIMAL as unscaled integers and DATE as days, as the batches hold them."""
    cols = []
    for name in table.column_names:
        c = table.column(name)
        if pa.types.is_decimal(c.type):
            c = pa.array([None if v is None else int(v.scaleb(c.type.scale)) for v in c.to_pylist()], pa.int64())
        elif pa.types.is_date32(c.type):
            c = c.cast(pa.int32())
        cols.append(c)
    return pa.table(cols, names=table.column_names)


def bloom_values(schema, batch, name):
    col = batch.value_column([f.name for f in schema.value_type.fields].index(name))
    return col.to_pylist()


def logical_of(schema, name):
    return next(f.type for f in schema.value_type.fields if f.name == name)


# ------------------------------------------------------------------------------------------------ one pipeline

def check(ok, what):
    assert ok, what


def pipeline(case: Case, from_device: bool, tmp: str) -> dict:
    """Decode -> deletion vector -> merge -> rebind + merge -> slices -> Arrow export -> Parquet and ORC encode -> bloom
    file index, every step checked against its reference.  Returns what it computed, for the comparison with the same
    pipeline on another thread."""
    schema, out = case.schema, {}
    open_sections = []

    def decode(sec):
        files = case.sections[sec]
        if from_device:
            up = FileUpload(files)
            try:
                readers, _ = read_section(schema, up.wait(), 3, file_format=case.formats[sec])
            finally:
                up.close()
        else:
            readers, _ = read_section(schema, files, 3, file_format=case.formats[sec])
        open_sections.append(readers)
        for r, rd in enumerate(readers):
            got = fetch_run(schema, rd._handle)
            check(got.equals(case.runs[sec][r]), f"{case.kind} section {sec} run {r}: {got.first_difference(case.runs[sec][r])}")
        return readers

    merge = None
    try:
        a = decode(0)
        dv = apply_deletion_vector(schema, a[0], case.deleted)
        open_sections.append([dv])
        got = fetch_run(schema, dv._handle)
        check(got.equals(case.after_dv), f"{case.kind} deletion vector: {got.first_difference(case.after_dv)}")
        merge = SortMergeReader([dv] + a[1:], case.spec)
        merge.readers = []                                  # (the sections are closed below)
        merge.execute()
        out["merged_a"] = got = merge.fetch()
        check(got.equals(case.want[0]), f"{case.kind} merge A: {got.first_difference(case.want[0])}")

        b = decode(1)
        merge.rebind(b)
        merge.readers = []
        merge.execute()
        out["merged_b"] = got = merge.fetch()
        want = case.want[1]
        check(got.equals(want), f"{case.kind} merge B: {got.first_difference(want)}")
        h = merge._merge_h

        out["slices"] = []
        for lo, hi in case.slices:
            s = fetch_slice(schema, h, lo, hi)
            check(s.equals(slice_rows(want, lo, hi)), f"{case.kind} slice {lo}:{hi}")
            out["slices"].append(s)
        out["exports"] = []
        for row0, n in case.exports:
            rb = export_arrow(schema, h, row0, n)
            g = arrow_to_batch(schema, pa.Table.from_batches([rb]))
            check(g.equals(slice_rows(want, row0, row0 + n)), f"{case.kind} export {row0}+{n}")
            out["exports"].append(g)

        row0, n = case.encoded
        part = slice_rows(want, row0, row0 + n)
        pq_path, orc_path = os.path.join(tmp, "out.parquet"), os.path.join(tmp, "out.orc")
        KeyValueDataFileWriter(schema, pq_path, level=1, compression="zstd", page_rows=1000, row_group_rows=4000,
                               page_index=True).write(h, row0, n)
        KeyValueDataFileWriter(schema, orc_path, level=1, file_format="orc", compression="zstd", stripe_rows=3000,
                               row_index_stride=1000, bloom_filter_columns=case.bloom,
                               bloom_filter_fpp=0.05).write(h, row0, n)
        out["parquet"], out["orc"] = open(pq_path, "rb").read(), open(orc_path, "rb").read()
        back = arrow_to_batch(schema, normalise(pq.read_table(io.BytesIO(out["parquet"]))))
        check(back.equals(part), f"{case.kind} Parquet file: {back.first_difference(part)}")
        back = arrow_to_batch(schema, normalise(porc.read_table(io.BytesIO(out["orc"]))))
        check(back.equals(part), f"{case.kind} ORC file: {back.first_difference(part)}")

        opts = {"file-index.bloom-filter.columns": ",".join(case.bloom)}
        opts.update({f"file-index.bloom-filter.{c}.items": "4000" for c in case.bloom})
        out["index"] = DataFileIndexWriter(schema, FileIndexOptions.from_options(opts)).build(h, row0, n)
        for c in case.bloom:
            want_filter = R.filter_of(logical_of(schema, c), bloom_values(schema, part, c), items=4000)
            check(out["index"][c] == want_filter, f"{case.kind} bloom filter of {c}")
    finally:
        if merge is not None:
            merge.close()
        for readers in open_sections:
            for rd in readers:
                rd.close()
    return out


def same_outputs(a: dict, b: dict, what: str):
    assert a.keys() == b.keys()
    for key in ("merged_a", "merged_b"):
        assert a[key].equals(b[key]), f"{what}: {key} {a[key].first_difference(b[key])}"
    for key in ("slices", "exports"):
        for x, y in zip(a[key], b[key]):
            assert x.equals(y), f"{what}: {key}"
    assert a["parquet"] == b["parquet"], f"{what}: the Parquet file differs from the single-threaded one"
    assert a["orc"] == b["orc"], f"{what}: the ORC file differs from the single-threaded one"
    assert a["index"] == b["index"], f"{what}: the file index differs from the single-threaded one"


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    tmp = str(tmp_path_factory.mktemp("concurrency_inputs"))
    N.init(0)
    return [Case(KIND_NAMES[w % len(KIND_NAMES)], 31 + w, w // len(KIND_NAMES), tmp) for w in range(WORKERS)]


def run_threads(fns):
    """Runs fns[i]() on thread i, all started together; re-raises the first failure."""
    errors = [None] * len(fns)
    start = threading.Barrier(len(fns))

    def body(i):
        try:
            start.wait()
            fns[i]()
        except BaseException as e:                # noqa: B902 - surfaced below
            errors[i] = e
    th = [threading.Thread(target=body, args=(i,)) for i in range(len(fns))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for e in errors:
        if e is not None:
            raise e


def test_concurrent_pipelines_equal_the_single_threaded_ones(cases, tmp_path):
    """8 workers, 2 rounds, a dirty cache before each round (and before each single-threaded pass): round 0 decodes from
    host bytes and round 1 from uploaded device bytes; every file, batch and filter equals the single-threaded one."""
    base = []
    for w, case in enumerate(cases):
        dirty_cache(copies=1)
        d = tmp_path / f"single{w}"
        d.mkdir()
        base.append(pipeline(case, from_device=False, tmp=str(d)))
    compared = {"files": 0, "batches": 0}
    for rnd in range(ROUNDS):
        dirty_cache()
        results = [None] * WORKERS

        def work(w, rnd=rnd):
            d = tmp_path / f"r{rnd}w{w}"
            d.mkdir()
            results[w] = pipeline(cases[w], from_device=rnd % 2 == 1, tmp=str(d))
        run_threads([lambda w=w: work(w) for w in range(WORKERS)])
        for w in range(WORKERS):
            same_outputs(results[w], base[w], f"round {rnd} worker {w} ({cases[w].kind})")
            compared["files"] += 2
            compared["batches"] += 2 + len(results[w]["slices"]) + len(results[w]["exports"])
    print(f"compared with the single-threaded pass: {compared['files']} files, {compared['batches']} batches")
    assert compared == {"files": 2 * WORKERS * ROUNDS, "batches": 9 * WORKERS * ROUNDS}


# ------------------------------------------------------------------------------------------------ handoffs

def test_decode_merge_export_and_free_on_different_threads(cases):
    """Decode on thread A, merge on B, export on C, free every handle on D; B to D never called pg_init (the calls bind
    the device themselves, and ~Merge runs on D)."""
    case = cases[0]
    schema = case.schema
    dirty_cache(copies=1)
    box = {}

    def on(fn):
        t = threading.Thread(target=fn)
        t.start()
        t.join()

    on(lambda: box.update(readers=read_section(schema, case.sections[1], 3, file_format=case.formats[1])[0]))
    assert "readers" in box

    def merge():
        rd = SortMergeReader.create_sort_merge_reader(box["readers"], None, None, case.spec)
        rd.execute()
        box["merge"] = rd
    on(merge)
    on(lambda: box.update(batch=export_arrow(schema, box["merge"]._merge_h)))
    on(lambda: box["merge"].close())
    got = arrow_to_batch(schema, pa.Table.from_batches([box["batch"]]))
    assert got.equals(case.want[1]), got.first_difference(case.want[1])


def test_upload_next_section_while_another_thread_decodes(cases):
    """INTEGRATION.md's pipeline: the upload of section i + 1 starts on one thread while another decodes and merges
    section i from its device bytes."""
    sections = [(c.sections[s], c.formats[s], c.runs[s], c) for c in cases[:4] for s in range(2)]
    dirty_cache(copies=2)
    ups = [FileUpload(sections[0][0])]
    for i, (files, fmt, runs, case) in enumerate(sections):
        box = {}

        def upload(i=i):
            if i + 1 < len(sections):
                ups.append(FileUpload(sections[i + 1][0]))

        def decode(i=i, fmt=fmt, case=case):
            readers, _ = read_section(case.schema, ups[i].wait(), 3, file_format=fmt)
            try:
                box["got"] = merge_readers(case, readers)
            finally:
                for r in readers:
                    r.close()
        run_threads([upload, decode])
        ups[i].close()
        want = pyoracle.merge(case.schema, case.spec, runs)
        assert box["got"].equals(want), (i, box["got"].first_difference(want))


def merge_readers(case, readers):
    rd = SortMergeReader.create_sort_merge_reader(readers, None, None, case.spec)
    rd.readers = []
    try:
        rd.execute()
        return rd.fetch()
    finally:
        rd.close()


# ------------------------------------------------------------------------------------------------ free while in use

ATTEMPTS = 6


def encode_bytes(schema, handle):
    """pg_parquet_encode of a whole run or merge batch, one call on `handle`, and the file's bytes."""
    lib = N.load()
    names = file_column_names(schema)
    arr = (C.c_char_p * len(names))(*[x.encode() for x in names])
    opts, fh = N.PgParquetWriteOptions(0, 1000, 0), C.c_uint64(0)
    N.check(lib.pg_parquet_encode(handle, arr, 0, -1, C.byref(opts), C.byref(fh)))
    try:
        meta = N.PgFileMeta()
        N.check(lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
        buf = np.empty(max(meta.file_bytes, 1), np.uint8)
        N.check(lib.pg_parquet_file_fetch(fh.value, buf.ctypes.data, meta.file_bytes))
        return buf[: meta.file_bytes].tobytes()
    finally:
        lib.pg_parquet_file_free(fh.value)


def test_free_while_another_thread_is_inside_a_call(cases):
    """A run, a view or a merge handle freed while another thread is inside pg_export_arrow, pg_run_fetch, pg_run_slice
    or pg_parquet_encode on it: the call returns the right result or PG_ERR_INVALID ('unknown ... handle'), never wrong
    data.  A fixed number of attempts per call, half of them with the free started first.

    Each call is one entry point on the handle, as the contract reads (the call finishes on the object it found).  A
    view of a merge batch does not keep the merge (include/paimon_gpu.h), so for a merge only pg_run_slice's own
    result is checked (the view's row count), not rows read through the view after the merge may be gone."""
    case = cases[0]
    schema, lib = case.schema, N.load()
    run_batch = case.runs[1][0]
    outcomes = {"ok": 0, "refused": 0}

    def fresh(kind):
        """-> (a handle, the batch it holds, what closes the rest)"""
        if kind == "merge":
            rd = SortedRunReader(schema, run_batch)
            m = SortMergeReader([rd], case.spec)
            m.readers = []
            m.execute()
            lib.pg_run_free(rd._handle)
            return m._merge_h, pyoracle.merge(schema, case.spec, [run_batch]), [m.close]
        sh = _SchemaHandle(schema, 0)
        h = SortedRunReader(schema, run_batch)._open(sh.handle)
        if kind == "run":
            return h, run_batch, [sh.close]
        v, start = C.c_uint64(0), C.c_int64(0)
        N.check(lib.pg_run_slice(h, 256, run_batch.n_rows, C.byref(v), C.byref(start)))
        lib.pg_run_free(h)
        return v.value, slice_rows(run_batch, 256, run_batch.n_rows), [sh.close]

    want_file = {}
    for kind in ("run", "view", "merge"):                # the files of the three sources, encoded without a race
        handle, want, closers = fresh(kind)
        want_file[kind] = encode_bytes(schema, handle)
        back = arrow_to_batch(schema, normalise(pq.read_table(io.BytesIO(want_file[kind]))))
        assert back.equals(want), back.first_difference(want)
        lib.pg_merge_free(handle) if kind == "merge" else lib.pg_run_free(handle)
        for c in closers:
            c()

    def call(kind, op, handle, want):
        """One entry point on `handle`; -> a check of its result, to run after both threads are done"""
        if op == "export":
            rb = export_arrow(schema, handle)
            return lambda: check(arrow_to_batch(schema, pa.Table.from_batches([rb])).equals(want), "export")
        if op == "fetch":
            got = fetch_run(schema, handle)
            return lambda: check(got.equals(want), "fetch")
        if op == "slice":
            v, start = C.c_uint64(0), C.c_int64(0)
            N.check(lib.pg_run_slice(handle, 131, want.n_rows - 5, C.byref(v), C.byref(start)))
            try:
                rows = C.c_int64(0)
                N.check(lib.pg_run_layout(v.value, C.byref(rows), None, None, schema.n_cols))
                got = None if kind == "merge" else fetch_run(schema, v.value)   # (a view of a run keeps the run)
            finally:
                lib.pg_run_free(v.value)
            assert start.value == 3 and rows.value == want.n_rows - 5 - 128
            return lambda: got is None or check(slice_rows(got, 3, rows.value).equals(slice_rows(want, 131, want.n_rows - 5)),
                                                "slice")
        data = encode_bytes(schema, handle)
        return lambda: check(data == want_file[kind], "encode")

    calls = [(kind, op) for kind in ("run", "view", "merge") for op in ("export", "fetch", "slice", "encode")
             if not (kind == "merge" and op == "fetch")]              # (pg_run_fetch takes runs and views)
    for kind, op in calls:
        for attempt in range(ATTEMPTS):
            dirty_cache(copies=2)
            handle, want, closers = fresh(kind)
            box = {"err": None, "verify": None}

            def use():
                try:
                    box["verify"] = call(kind, op, handle, want)
                except N.PaimonGpuError as e:
                    box["err"] = e

            def free():
                lib.pg_merge_free(handle) if kind == "merge" else lib.pg_run_free(handle)
            run_threads([use, free] if attempt % 2 == 0 else [free, use])
            if box["err"] is None:
                box["verify"]()
                outcomes["ok"] += 1
            else:
                err = box["err"]
                assert err.status == 1 and "unknown" in err.message, (kind, op, attempt, err)
                outcomes["refused"] += 1
            for c in closers:
                c()
    assert outcomes["ok"] + outcomes["refused"] == len(calls) * ATTEMPTS
    print(f"free while in use: {outcomes}")


# ------------------------------------------------------------------------------------------------ range streaming

def test_range_streaming_over_a_wide_schema_with_a_dirty_cache():
    schema = datagen.schema_c3(n_i64=6, n_f64=4, n_str=6)
    runs = datagen.make_runs(schema, 6, 120_000, seed=3, null_prob=0.35)
    spec = PartialUpdateMergeFunction.factory({}, schema.value_type, ["pk"]).create()
    want = merge_runs(schema, spec, runs)
    dirty_cache()
    rd = RangeStreamingMergeReader(schema, runs, spec, target_rows=9_000, depth=4)
    try:
        batches = []
        while (b := rd.read_batch()) is not None:
            batches.append(b)
    finally:
        rd.close()
    assert len(batches) > 8
    got = concat_batches(schema, batches)
    assert got.equals(want), got.first_difference(want)
    assert got.equals(pyoracle.merge(schema, spec, runs))


# ------------------------------------------------------------------------------------------------ pinned ring growth

def rss_bytes():
    with open("/proc/self/statm") as f:
        return int(f.read().split()[1]) * os.sysconf("SC_PAGE_SIZE")


def test_merge_handles_do_not_accumulate_pinned_host_memory():
    """Every merge handle stages its descriptors through an 8 MiB page-locked ring; 64 handles opened, executed and
    freed on one long-lived thread, then on 16 short-lived threads, must give that memory back."""
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=1)
    runs = datagen.make_runs(schema, 3, 3000, seed=4, null_prob=0.2)
    spec = DeduplicateMergeFunction.factory().create()
    want = pyoracle.merge(schema, spec, runs)

    def merges(n):
        for _ in range(n):
            got = merge_runs(schema, spec, runs)
            assert got.equals(want)
    merges(2)                                            # one-time allocations of the thread and the process
    before = rss_bytes()
    merges(64)
    one_thread = rss_bytes() - before
    before = rss_bytes()
    for _ in range(4):
        th = [threading.Thread(target=merges, args=(1,)) for _ in range(16)]
        for t in th:
            t.start()
        for t in th:
            t.join()
    short_lived = rss_bytes() - before
    print(f"RSS growth over 64 merge handles: one thread {one_thread >> 20} MiB, "
          f"64 short-lived threads {short_lived >> 20} MiB")
    assert one_thread < 64 * (8 << 20) // 8, one_thread
    assert short_lived < 64 * (8 << 20) // 8, short_lived


# ------------------------------------------------------------------------------------------------ one path at a time

def host_run_batch(n, seed, run_index=0):
    schema = all_types_schema()
    keys = np.arange(n, dtype=np.int64) * 5 + 1
    run = datagen.make_run(schema, run_index, keys, seed, null_prob=0.4)
    return schema, decimal_schema_runs(schema, [run], ("dec",))[0]


def single_path(path, tmp):
    """One device path on a dirty cache, against its reference."""
    if path.startswith("parquet_decode") or path.startswith("orc_decode"):
        schema = all_types_schema()
        batch = host_run_batch(7001, 9)[1]
        if path.startswith("parquet_decode"):
            data = parquet_bytes(batch, PARQUET_OPTS[int(path.rsplit("_", 1)[1])])
            readers, _ = read_section(schema, [(data, 0)], 1)
        else:
            codec, version = path.split(":")[1:]
            t = normalise(to_arrow(batch))
            t = t.set_column(t.column_names.index("dt"), "dt", t.column("dt").cast(pa.date32()))
            buf = io.BytesIO()
            porc.write_table(t, buf, compression=codec, file_version=version, stripe_size=64 * 1024)
            readers, _ = read_section(schema, [(buf.getvalue(), 0)], 1, file_format="orc")
        try:
            got = fetch_run(schema, readers[0]._handle)
        finally:
            readers[0].close()
        assert got.equals(batch), got.first_difference(batch)
        return
    if path.startswith("host_run"):
        n = int(path.split(":")[1])
        schema, batch = host_run_batch(n, n)
        spec = DeduplicateMergeFunction.factory().create()
        other = host_run_batch(n, n + 1, run_index=1)[1]
        # a second run of the same keys: the merge reads the first one's validity and var-len tails in whole words
        got = merge_runs(schema, spec, [batch, other])
        assert got.equals(pyoracle.merge(schema, spec, [batch, other]))
        rd = SortedRunReader(schema, batch)
        sh = _SchemaHandle(schema, 0)
        try:
            h = rd._open(sh.handle)
            back = fetch_run(schema, h)
            assert back.equals(batch), back.first_difference(batch)
            for row0, k in ((0, n), (1, n - 1), (n // 2, n - n // 2)):
                if k > 0:
                    g = arrow_to_batch(schema, pa.Table.from_batches([export_arrow(schema, h, row0, k)]))
                    assert g.equals(slice_rows(batch, row0, row0 + k)), (row0, k)
            pth = os.path.join(tmp, "h.parquet")
            KeyValueDataFileWriter(schema, pth, level=1, page_rows=37, page_index=True).write(h)
            back = arrow_to_batch(schema, normalise(pq.read_table(pth)))
            assert back.equals(batch), back.first_difference(batch)
        finally:
            rd.close()
            sh.close()
        return
    case_kind = {"deletion_vector": "all_types_dedup", "parquet_encode": "c3_partial_update", "orc_encode": "all_types_dedup",
                 "file_index": "composite_key_dedup", "arrow_export": "composite_key_dedup"}.get(path)
    if path.startswith("merge_"):
        engine = path.split("_", 1)[1]
        schema = all_types_schema()
        runs = [host_run_batch(2000 + 37 * r, 50 + r, run_index=r)[1] for r in range(4)]
        spec = {"dedup": DeduplicateMergeFunction.factory().create(),
                "partial_update": PartialUpdateMergeFunction.factory({}, schema.value_type, ["pk"]).create(),
                "first_row": FirstRowMergeFunction.factory().create(),
                "aggregate": AggregateMergeFunction.factory(AGG_OPTIONS_ALL, schema.value_type, ["pk"]).create()}[engine]
        got = merge_runs(schema, spec, runs)
        want = pyoracle.merge(schema, spec, runs)
        assert got.equals(want), got.first_difference(want)
        return
    case = Case(case_kind, 77, 1 if path == "orc_encode" else 0, tmp)
    pipeline(case, from_device=path == "orc_encode", tmp=tmp)


AGG_OPTIONS_ALL = {"fields.l.aggregate-function": "max", "fields.i.aggregate-function": "min",
                   "fields.dt.aggregate-function": "max", "fields.dec.aggregate-function": "sum",
                   "fields.d.aggregate-function": "max", "fields.s.aggregate-function": "last_non_null_value",
                   "fields.bin.aggregate-function": "first_non_null_value"}
SINGLE_PATHS = ([f"parquet_decode_{i}" for i in range(len(PARQUET_OPTS))] +
                [f"orc_decode:{c}:{v}" for c in ("uncompressed", "zlib", "zstd", "lz4") for v in ("0.12",)] +
                ["orc_decode:zlib:0.11", "orc_decode:uncompressed:0.11", "deletion_vector"] +
                [f"merge_{e}" for e in ("dedup", "partial_update", "first_row", "aggregate")] +
                ["parquet_encode", "orc_encode", "file_index", "arrow_export"] +
                [f"host_run:{n}" for n in (1, 7, 9, 33, 127, 129, 1001, 4099)])


@pytest.mark.parametrize("path", SINGLE_PATHS)
def test_dirty_cache_single_thread(path, tmp_path):
    """Each device path once, every buffer it takes from a cache filled with 0xA5 bytes; host runs of row counts that
    are not multiples of 8, 32 or 128 reach the validity and read-past tails that pg_run_open does not copy."""
    dirty_cache(copies=2)
    single_path(path, str(tmp_path))
