"""Host-side mirror of the reference's reader interfaces for the merge path.

  RecordReader            paimon-common/src/main/java/org/apache/paimon/reader/RecordReader.java:40-72
  SortMergeReader         paimon-core/.../mergetree/compact/SortMergeReader.java:41-57
  ReducerMergeFunctionWrapper  …/compact/ReducerMergeFunctionWrapper.java:45-73 (semantics live in the plan kernel)
  DropDeleteReader        paimon-core/.../mergetree/DropDeleteReader.java:50-68
  MergeTreeReaders.readerForSection  paimon-core/.../mergetree/MergeTreeReaders.java:67-92

Same names, same argument meaning, same error behaviour (the exceptions carry the reference's
messages), but batches are columnar (``KeyValueBatch``) instead of row iterators, and all work
happens in libpaimon_gpu.so.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from . import _native as N
from .columnar import Column, KeyValueBatch
from .merge_function import MergeSpec, SortEngine
from .types import KeyValueSchema, PhysicalType, is_varlen, numpy_dtype


def _np_ptr(a: Optional[np.ndarray]) -> Optional[int]:
    return None if a is None else a.ctypes.data


class _SchemaHandle:
    def __init__(self, schema: KeyValueSchema, device: int):
        self.schema = schema
        lib = N.init(device)
        kf = (N.PgField * schema.n_key)(*[N.PgField(int(f.physical), 0) for f in schema.key_type.fields])
        vf = (N.PgField * max(schema.n_val, 1))(
            *[N.PgField(int(f.physical), int(f.nullable)) for f in schema.value_type.fields])
        desc = N.PgSchemaDesc(schema.n_key, schema.n_val, kf, vf)
        h = C.c_uint64(0)
        N.check(lib.pg_schema_create(C.byref(desc), C.byref(h)))
        self.handle = h.value

    def close(self):
        if self.handle:
            N.load().pg_schema_free(self.handle)
            self.handle = 0


class RecordReader:
    """RecordReader<KeyValue>: read_batch() returns a columnar batch or None at end of input."""

    def read_batch(self) -> Optional[KeyValueBatch]:
        raise NotImplementedError

    def close(self) -> None:
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


@dataclass
class DeviceColumn:
    data: int
    offsets: int = 0
    validity: int = 0


class SortedRunReader(RecordReader):
    """One sorted run (keys strictly increasing) — what MergeTreeReaders.readerForRun yields
    (MergeTreeReaders.java:94-101).  Either host columns (copied to the device when the merge opens
    it) or device-resident columns (pointers borrowed; `keepalive` pins their owner)."""

    def __init__(self, schema: KeyValueSchema, batch: Optional[KeyValueBatch] = None, *,
                 n_rows: Optional[int] = None, device_columns: Optional[Sequence[DeviceColumn]] = None,
                 keepalive=None):
        self.schema = schema
        self.batch = batch
        self.device_columns = list(device_columns) if device_columns is not None else None
        self.n_rows = batch.n_rows if batch is not None else int(n_rows or 0)
        self.keepalive = keepalive
        self._consumed = False
        self._handle = 0

    @staticmethod
    def from_device(schema: KeyValueSchema, n_rows: int, columns: Sequence[DeviceColumn], keepalive=None):
        return SortedRunReader(schema, None, n_rows=n_rows, device_columns=columns, keepalive=keepalive)

    @staticmethod
    def from_native_run(schema: KeyValueSchema, n_rows: int, run_handle: int, keepalive=None):
        """A run that already lives in the library (e.g. decoded from a Parquet file on the device)."""
        r = SortedRunReader(schema, None, n_rows=n_rows, keepalive=keepalive)
        r._handle = run_handle
        r._native = True
        return r

    def read_batch(self) -> Optional[KeyValueBatch]:
        if self._consumed:
            return None
        self._consumed = True
        if self.batch is not None:
            return self.batch
        if getattr(self, "_native", False) and self._handle:
            return fetch_run(self.schema, self._handle)
        return None

    # -- native registration (used by SortMergeReader) --
    def _open(self, schema_handle: int) -> int:
        if getattr(self, "_native", False):
            return self._handle
        lib = N.load()
        nc = self.schema.n_cols
        cols = (N.PgColumn * nc)()
        keep = []
        if self.device_columns is not None:
            for i, dc in enumerate(self.device_columns):
                cols[i] = N.PgColumn(dc.data or None, dc.offsets or None, dc.validity or None)
            mem = N.PG_MEM_DEVICE
        else:
            for i, col in enumerate(self.batch.columns):
                data = np.ascontiguousarray(col.data)
                offs = None if col.offsets is None else np.ascontiguousarray(col.offsets, np.int32)
                val = None if col.valid is None else np.ascontiguousarray(col.valid, np.uint8)
                keep += [data, offs, val]
                cols[i] = N.PgColumn(_np_ptr(data), _np_ptr(offs), _np_ptr(val))
            mem = N.PG_MEM_HOST
        desc = N.PgRunDesc(self.n_rows, cols)
        h = C.c_uint64(0)
        N.check(lib.pg_run_open(schema_handle, C.byref(desc), mem, C.byref(h)))
        self._handle = h.value
        return self._handle

    def close(self) -> None:
        if self._handle:
            N.load().pg_run_free(self._handle)
            self._handle = 0


def apply_deletion_vector(schema: KeyValueSchema, reader: "SortedRunReader", deleted_positions, schema_handle: int = 0,
                          device: int = 0) -> "SortedRunReader":
    """ApplyDeletionVectorReader (paimon-core/.../deletionvectors/ApplyDeletionVectorReader.java:31-54): the run
    without the rows whose file position is in `deleted_positions` (an iterable of row ordinals — what
    DeletionVector.isDeleted answers — or a ready LSB-first bitmap as np.uint8).  Runs on the device."""
    lib = N.init(device)
    own = None
    if not reader._handle:
        own = _SchemaHandle(schema, device)
        reader._open(own.handle)
    try:
        if isinstance(deleted_positions, np.ndarray) and deleted_positions.dtype == np.uint8:
            bitmap = np.ascontiguousarray(deleted_positions)
            n_bits = len(bitmap) * 8
        else:
            pos = np.asarray(sorted(set(int(p) for p in deleted_positions)), np.int64)
            n_bits = int(pos[-1]) + 1 if len(pos) else 0
            flags = np.zeros(n_bits, bool)
            flags[pos] = True
            bitmap = np.packbits(flags, bitorder="little") if n_bits else np.zeros(1, np.uint8)
        h = C.c_uint64(0)
        N.check(lib.pg_run_apply_deletion_vector(reader._handle, bitmap.ctypes.data, n_bits, C.byref(h)))
        n_rows = C.c_int64(0)
        N.check(lib.pg_run_layout(h.value, C.byref(n_rows), None, None, schema.n_cols))
        return SortedRunReader.from_native_run(schema, int(n_rows.value), h.value, keepalive=None)
    finally:
        if own is not None:
            own.close()


def fetch_run(schema: KeyValueSchema, run_handle: int) -> KeyValueBatch:
    """Device-resident run -> host columns (pg_run_layout + pg_run_fetch)."""
    lib = N.load()
    nc = schema.n_cols
    n_rows = C.c_int64(0)
    data_bytes = np.zeros(nc, np.int64)
    has_valid = np.zeros(nc, np.int32)
    N.check(lib.pg_run_layout(run_handle, C.byref(n_rows), data_bytes.ctypes.data, has_valid.ctypes.data, nc))
    n = n_rows.value
    host = (N.PgOutColumn * nc)()
    cols: List[Column] = []
    for i, t in enumerate(schema.physical_types()):
        if data_bytes[i] < 0:                               # the run was decoded without this column (projection)
            host[i] = N.PgOutColumn(None, None, None, 0)
            cols.append(None)
            continue
        valid = np.zeros((n + 7) // 8 + 8, np.uint8) if has_valid[i] else None
        if is_varlen(t):
            data = np.zeros(max(int(data_bytes[i]), 1), np.uint8)
            offs = np.zeros(n + 1, np.int32)
            host[i] = N.PgOutColumn(_np_ptr(data), _np_ptr(offs), _np_ptr(valid), int(data_bytes[i]))
            cols.append(Column(t, data[: int(data_bytes[i])], offs, valid))
        else:
            data = np.zeros(max(n, 1), numpy_dtype(t))
            host[i] = N.PgOutColumn(_np_ptr(data), None, _np_ptr(valid), int(data_bytes[i]))
            cols.append(Column(t, data[:n], None, valid))
    N.check(lib.pg_run_fetch(run_handle, host, nc))
    for col in cols:                                  # a view (pg_run_slice) keeps the source's absolute offsets
        if col is not None and col.offsets is not None and n > 0 and col.offsets[0] != 0:
            col.offsets -= col.offsets[0]
    return KeyValueBatch(schema, cols)


def slice_rows(batch: KeyValueBatch, lo: int, hi: int) -> KeyValueBatch:
    """Rows [lo, hi) of a host batch (copies)."""
    from .columnar import pack_validity, unpack_validity
    cols = []
    for col in batch.columns:
        if col is None:
            cols.append(None)
            continue
        valid = None
        if col.valid is not None:
            valid = pack_validity(unpack_validity(col.valid, len(col))[lo:hi])
        if col.offsets is not None:
            o = np.asarray(col.offsets[lo:hi + 1], np.int64)
            data = np.array(col.data[int(o[0]):int(o[-1])], copy=True) if hi > lo else np.zeros(0, np.uint8)
            cols.append(Column(col.type, data, (o - (o[0] if hi > lo else 0)).astype(np.int32) if hi > lo
                               else np.zeros(1, np.int32), valid))
        else:
            cols.append(Column(col.type, np.array(col.data[lo:hi], copy=True), None, valid))
    return KeyValueBatch(batch.schema, cols)


def export_arrow(schema: KeyValueSchema, source_handle: int, row0: int = 0, n_rows: int = -1):
    """Rows of a merge handle's batch (or of a run) through the Arrow C Data Interface (pg_export_arrow), imported
    with pyarrow exactly as the Java side imports them with org.apache.arrow.c.Data.importVectorSchemaRoot: a
    pyarrow.RecordBatch whose columns carry the Paimon file field names.  The buffers are page-locked host memory
    owned by the batch and released with it."""
    import pyarrow as pa
    from pyarrow.cffi import ffi
    lib = N.load()
    names = [f.name for f in schema.file_fields()]
    arr = (C.c_char_p * len(names))(*[nm.encode() for nm in names])
    c_schema = ffi.new("struct ArrowSchema*")
    c_array = ffi.new("struct ArrowArray*")
    N.check(lib.pg_export_arrow(source_handle, arr, row0, n_rows, int(ffi.cast("uintptr_t", c_array)),
                                int(ffi.cast("uintptr_t", c_schema))))
    return pa.RecordBatch._import_from_c(int(ffi.cast("uintptr_t", c_array)), int(ffi.cast("uintptr_t", c_schema)))


def fetch_slice(schema: KeyValueSchema, source_handle: int, lo: int, hi: int) -> KeyValueBatch:
    """Rows [lo, hi) of a device-resident run, or of a merge handle's current batch, as host columns
    (pg_run_slice view + pg_run_fetch)."""
    lib = N.load()
    h, start = C.c_uint64(0), C.c_int64(0)
    N.check(lib.pg_run_slice(source_handle, lo, hi, C.byref(h), C.byref(start)))
    try:
        view = fetch_run(schema, h.value)
    finally:
        lib.pg_run_free(h.value)
    return slice_rows(view, int(start.value), int(start.value) + (hi - lo))


@dataclass
class DeviceBatch:
    """The merged batch left on the device: (data, offsets, validity, data_bytes) pointers per column."""
    n_rows: int
    columns: List[N.PgOutColumn]


class SortMergeReader(RecordReader):
    """k-way merge of sorted runs + per-key merge function (+ optional DropDeleteReader).

    Like SortMergeReaderWithLoserTree (SortMergeReaderWithLoserTree.java:67-73) the reader produces
    exactly one batch."""

    @staticmethod
    def create_sort_merge_reader(readers: Sequence[SortedRunReader], user_key_comparator=None,
                                 user_defined_seq_comparator=None,
                                 merge_function_wrapper: Optional[MergeSpec] = None,
                                 sort_engine: SortEngine = SortEngine.LOSER_TREE,
                                 device: int = 0) -> "SortMergeReader":
        """SortMergeReader.createSortMergeReader (SortMergeReader.java:41-57).

        `user_key_comparator` must be None (the key order is the schema's natural order, which is what
        the reference's generated comparator implements); `user_defined_seq_comparator` is a list of
        value-field indexes or None; `merge_function_wrapper` is the MergeSpec built by a
        MergeFunctionFactory.  `sort_engine` is accepted for signature parity: both engines produce the
        same rows and the device implements one algorithm."""
        if user_key_comparator is not None:
            raise N.UnsupportedOnDevice(2, "custom key comparators cannot run on the device")
        if merge_function_wrapper is None:
            raise ValueError("merge_function_wrapper (MergeSpec) is required")
        spec = merge_function_wrapper
        if user_defined_seq_comparator is not None:
            if hasattr(user_defined_seq_comparator, "apply"):           # UserDefinedSeqComparator
                spec = user_defined_seq_comparator.apply(spec)
            else:                                                       # plain list of value-field indexes
                spec = spec.normalised(readers[0].schema.n_val) if readers else spec
                spec.seq_fields = list(user_defined_seq_comparator)
        return SortMergeReader(list(readers), spec, None, device)

    def __init__(self, readers: List[SortedRunReader], spec: MergeSpec, seq_fields=None, device: int = 0,
                 start_rows: Optional[Sequence[int]] = None, schema: Optional[KeyValueSchema] = None):
        self.readers = readers
        self.lib = N.init(device)
        schema = readers[0].schema if readers else schema
        self.schema = schema
        self._done = False
        self._schema_h = None
        self._spec_h = 0
        self._merge_h = 0
        self._keep = []
        if schema is None:
            return
        self._schema_h = _SchemaHandle(schema, device)
        sp = spec.normalised(schema.n_val)
        seq = list(seq_fields) if seq_fields else list(sp.seq_fields)
        seq_arr = np.array(seq, np.int32)
        agg = np.array([int(a) for a in sp.agg], np.int32)
        ign = np.array([1 if b else 0 for b in sp.ignore_retract], np.uint8)
        self._keep += [seq_arr, agg, ign]
        gstart = np.zeros(len(sp.groups) + 1, np.int32)
        gfields = np.array([f for g in sp.groups for f in g] or [0], np.int32)
        for i, g in enumerate(sp.groups):
            gstart[i + 1] = gstart[i] + len(g)
        fgroup = np.array(sp.field_group, np.int32)
        gpd = np.array([1 if b else 0 for b in sp.group_partial_delete], np.uint8)
        rf = np.array([1 if b else 0 for b in sp.read_fields], np.uint8) if sp.read_fields else None
        self._read_fields = list(sp.read_fields) if sp.read_fields else None
        dec = np.array(sp.decimal, np.int32) if sp.decimal else None
        self._keep += [gstart, gfields, fgroup, gpd, rf, dec]
        has_groups = len(sp.groups) > 0
        cs = N.PgMergeSpec(int(sp.engine), int(sp.ignore_delete), int(sp.remove_record_on_delete),
                           int(sp.drop_delete), len(seq), _np_ptr(seq_arr) if len(seq) else None,
                           int(sp.seq_ascending), _np_ptr(agg), _np_ptr(ign), len(sp.groups),
                           _np_ptr(gstart) if has_groups else None, _np_ptr(gfields) if has_groups else None,
                           _np_ptr(fgroup) if has_groups else None, _np_ptr(gpd) if has_groups else None,
                           _np_ptr(rf), _np_ptr(dec))
        h = C.c_uint64(0)
        try:
            N.check(self.lib.pg_merge_spec_create(self._schema_h.handle, C.byref(cs), C.byref(h)))
            self._spec_h = h.value
            run_handles = (C.c_uint64 * max(len(readers), 1))()
            for i, r in enumerate(readers):
                run_handles[i] = r._open(self._schema_h.handle)
            mh = C.c_uint64(0)
            N.check(self.lib.pg_merge_open(self._spec_h, run_handles, len(readers), C.byref(mh)))
            self._merge_h = mh.value
            if start_rows is not None and any(start_rows):
                sr = np.array(list(start_rows), np.int64)
                N.check(self.lib.pg_merge_rebind(self._merge_h, run_handles, len(readers), _np_ptr(sr)))
        except Exception:
            self.close()
            raise

    def rebind(self, readers: List[SortedRunReader], start_rows: Optional[Sequence[int]] = None) -> None:
        """Same merge (schema, merge function, device arenas, stream) over other runs (pg_merge_rebind)."""
        self.readers = readers
        run_handles = (C.c_uint64 * max(len(readers), 1))()
        for i, r in enumerate(readers):
            run_handles[i] = r._open(self._schema_h.handle)
        sr = np.array(list(start_rows) if start_rows is not None else [0] * len(readers), np.int64)
        N.check(self.lib.pg_merge_rebind(self._merge_h, run_handles, len(readers), _np_ptr(sr)))

    # -- execution --
    def execute(self) -> None:
        N.check(self.lib.pg_merge_execute(self._merge_h))

    def stats(self) -> N.PgStats:
        st = N.PgStats()
        N.check(self.lib.pg_merge_stats(self._merge_h, C.byref(st)))
        return st

    def cuda_stream(self) -> int:
        p = C.c_void_p(0)
        N.check(self.lib.pg_merge_stream(self._merge_h, C.byref(p)))
        return p.value or 0

    def device_batch(self) -> DeviceBatch:
        b = N.PgBatch()
        N.check(self.lib.pg_merge_device_batch(self._merge_h, C.byref(b)))
        return DeviceBatch(b.n_rows, [b.cols[i] for i in range(b.n_cols)])

    def fetch(self, allocator=None) -> KeyValueBatch:
        """Device batch -> host columns (D2H).  `allocator(nbytes) -> np.uint8 array` lets the caller supply
        page-locked memory (the Java side passes direct buffers); default is ordinary numpy memory."""
        alloc = allocator or (lambda nbytes: np.zeros(nbytes, np.uint8))
        db = self.device_batch()
        n = db.n_rows
        types = self.schema.physical_types()
        host = (N.PgOutColumn * len(types))()
        cols: List[Column] = []
        nk2 = self.schema.n_key + 2
        for i, t in enumerate(types):
            oc = db.columns[i]
            if self._read_fields is not None and i >= nk2 and not self._read_fields[i - nk2]:
                host[i] = N.PgOutColumn(None, None, None, 0)       # not part of the read type
                cols.append(None)
                continue
            valid = alloc((n + 7) // 8 + 8) if oc.validity else None
            if is_varlen(t):
                data = alloc(max(int(oc.data_bytes), 1))
                offs = alloc(4 * (n + 1)).view(np.int32)
                host[i] = N.PgOutColumn(_np_ptr(data), _np_ptr(offs), _np_ptr(valid), oc.data_bytes)
                cols.append(Column(t, data[: int(oc.data_bytes)], offs, valid))
            else:
                dt = np.dtype(numpy_dtype(t))
                data = alloc(max(n, 1) * dt.itemsize).view(dt)
                host[i] = N.PgOutColumn(_np_ptr(data), None, _np_ptr(valid), oc.data_bytes)
                cols.append(Column(t, data[:n], None, valid))
        N.check(self.lib.pg_merge_fetch(self._merge_h, host, len(types)))
        return KeyValueBatch(self.schema, cols)

    def read_batch(self) -> Optional[KeyValueBatch]:
        if self._done or self.schema is None:
            return None
        self._done = True
        self.execute()
        batch = self.fetch()
        return batch if batch.n_rows > 0 else None

    def release_batch(self) -> None:
        if self._merge_h:
            self.lib.pg_merge_release(self._merge_h)

    def close(self) -> None:
        lib = N.load()
        if self._merge_h:
            lib.pg_merge_free(self._merge_h)
            self._merge_h = 0
        for r in self.readers:
            r.close()
        if self._spec_h:
            lib.pg_merge_spec_free(self._spec_h)
            self._spec_h = 0
        if self._schema_h is not None:
            self._schema_h.close()
            self._schema_h = None


def cut_key_ranges(keys: Sequence[np.ndarray], target_rows: int):
    """Cut k sorted key arrays into key ranges of about `target_rows` rows in total: a list of ranges, each a
    list of (lo, hi) row bounds per run.  Splitter keys are quantiles of a sample of all runs; a range holds
    every row whose key lies in [splitter[j-1], splitter[j])."""
    total = sum(len(k) for k in keys)
    n_ranges = max(1, -(-total // max(1, int(target_rows))))
    if n_ranges == 1 or total == 0:
        return [[(0, len(k)) for k in keys]]
    stride = max(1, total // (n_ranges * 64 * max(len(keys), 1)))
    sample = np.sort(np.concatenate([k[stride - 1::stride] for k in keys if len(k)]))
    if len(sample) == 0:
        return [[(0, len(k)) for k in keys]]
    cut_keys = np.unique(sample[(np.arange(1, n_ranges) * len(sample)) // n_ranges])
    cuts = [np.concatenate([[0], np.searchsorted(k, cut_keys, side="left"), [len(k)]]) for k in keys]
    return [[(int(c[j]), int(c[j + 1])) for c in cuts] for j in range(len(cut_keys) + 1)]


class RangeStreamingMergeReader(RecordReader):
    """Merge of HOST-resident sorted runs that flows through the device in key ranges.

    The reference's readers hand out one batch after the other (RecordReader.readBatch,
    paimon-common/.../reader/RecordReader.java:42-72; ConcatRecordReader.java:52-75 for key-disjoint pieces);
    here every batch is the merge of one key range of all runs.  The ranges are key-disjoint and ascending, so
    the concatenation of the batches equals the single batch SortMergeReader would produce.  `depth` ranges are
    in flight at a time, each on its own worker thread and CUDA stream: the host->device copy of range i+1
    overlaps the merge of range i and the device->host copy of range i-1 (PCIe is full duplex), and the device
    holds `depth` ranges instead of the whole bucket.

    Requires a single fixed-width integer primary-key column (the range cuts are binary searches on the host key
    arrays); other schemas use SortMergeReader."""

    def __init__(self, schema: KeyValueSchema, runs: Sequence[KeyValueBatch], spec: MergeSpec,
                 target_rows: int = 8 << 20, depth: int = 3, device: int = 0, allocator_factory=None):
        import threading
        self.schema = schema
        self.lib = N.init(device)
        self.runs = list(runs)
        self.spec = spec
        self.depth = max(1, depth)
        self.device = device
        self.allocator_factory = allocator_factory     # () -> allocator(nbytes) for one output batch
        if schema.n_key != 1 or is_varlen(schema.physical_types()[0]):
            raise N.UnsupportedOnDevice(2, "range streaming needs a single fixed-width integer key column")
        self.bytes_h2d = 0
        self.bytes_d2h = 0
        self.ranges = self._cut_ranges(max(1, int(target_rows)))
        self._tables = self._pointer_tables()
        self._results = {}
        self._errors = []
        self._cv = threading.Condition()
        self._next_out = 0
        self._consumed = 0
        self._closed = False
        self._threads = [threading.Thread(target=self._worker, args=(w,), daemon=True) for w in range(self.depth)]
        for t in self._threads:
            t.start()

    def _cut_ranges(self, target_rows: int):
        return cut_key_ranges([np.asarray(r.columns[0].data) for r in self.runs], target_rows)

    def _pointer_tables(self):
        """Per run: base address / element width of every column buffer, so that a range's pg_run_desc is a few
        vectorised operations (no per-column Python work on the hot path)."""
        tables = []
        for run in self.runs:
            nc = len(run.columns)
            data = np.zeros(nc, np.uint64); offs = np.zeros(nc, np.uint64); val = np.zeros(nc, np.uint64)
            width = np.zeros(nc, np.uint64)
            keep = []
            for i, col in enumerate(run.columns):
                d = np.ascontiguousarray(col.data)
                keep.append(d)
                data[i] = d.ctypes.data
                if col.offsets is not None:
                    o = np.ascontiguousarray(col.offsets, np.int32)
                    keep.append(o)
                    offs[i] = o.ctypes.data
                else:
                    width[i] = d.dtype.itemsize
                if col.valid is not None:
                    v = np.ascontiguousarray(col.valid, np.uint8)
                    keep.append(v)
                    val[i] = v.ctypes.data
            tables.append((data, offs, val, width, keep))
        return tables

    def _open_range(self, schema_handle: int, r: int, lo: int, hi: int):
        """Rows [lo, hi) of run r as a device run that starts at the 8-row boundary below lo (validity bitmaps
        are byte-granular); var-len columns keep absolute offsets and the whole payload as `data`
        (pg_run_open copies [offsets[0], offsets[n])).  Returns (run handle, start row)."""
        data, offs, val, width, _ = self._tables[r]
        lo8 = lo & ~7
        arr = np.empty((len(data), 3), np.uint64)
        arr[:, 0] = data + width * np.uint64(lo8)
        arr[:, 1] = np.where(offs != 0, offs + np.uint64(4 * lo8), 0)
        arr[:, 2] = np.where(val != 0, val + np.uint64(lo8 // 8), 0)
        cols = (N.PgColumn * len(data)).from_buffer(arr)
        desc = N.PgRunDesc(hi - lo8, cols)
        h = C.c_uint64(0)
        N.check(self.lib.pg_run_open(schema_handle, C.byref(desc), N.PG_MEM_HOST, C.byref(h)))
        return h.value, lo - lo8

    def _worker(self, w: int):
        rd = None
        k = len(self.runs)
        try:
            for j in range(w, len(self.ranges), self.depth):
                with self._cv:                          # bounded look-ahead: at most `depth` batches not yet consumed
                    while not self._closed and j >= self._consumed + self.depth:
                        self._cv.wait()
                    if self._closed:
                        return
                if rd is None:
                    rd = SortMergeReader([], self.spec, None, self.device, schema=self.schema)
                handles = (C.c_uint64 * max(k, 1))()
                starts = np.zeros(max(k, 1), np.int64)
                try:
                    for r, (lo, hi) in enumerate(self.ranges[j]):
                        handles[r], starts[r] = self._open_range(rd._schema_h.handle, r, lo, hi)
                    N.check(self.lib.pg_merge_rebind(rd._merge_h, handles, k, _np_ptr(starts)))
                    rd.execute()
                    alloc = self.allocator_factory() if self.allocator_factory else None
                    out = rd.fetch(allocator=alloc)
                    st = rd.stats()
                finally:
                    for r in range(k):
                        if handles[r]:
                            self.lib.pg_run_free(handles[r])
                with self._cv:
                    self.bytes_h2d += st.bytes_h2d
                    self.bytes_d2h += st.bytes_d2h
                    self._results[j] = out
                    self._cv.notify_all()
        except BaseException as e:                      # surfaced by read_batch
            with self._cv:
                self._errors.append(e)
                self._cv.notify_all()
        finally:
            if rd is not None:
                rd.close()

    def read_batch(self) -> Optional[KeyValueBatch]:
        while True:
            with self._cv:
                j = self._next_out
                if j >= len(self.ranges):
                    return None
                while j not in self._results and not self._errors:
                    self._cv.wait()
                if self._errors:
                    raise self._errors[0]
                out = self._results.pop(j)
                self._next_out += 1
                self._consumed += 1
                self._cv.notify_all()
            if out.n_rows > 0:
                return out

    def close(self) -> None:
        with self._cv:
            self._closed = True
            self._cv.notify_all()
        for t in self._threads:
            t.join()


def merge_runs(schema: KeyValueSchema, spec: MergeSpec, runs: Sequence[KeyValueBatch], device: int = 0) -> KeyValueBatch:
    """Convenience: merge host batches and return the (possibly empty) merged batch."""
    readers = [SortedRunReader(schema, b) for b in runs]
    if not readers:
        return KeyValueBatch.from_rows(schema, [])
    rd = SortMergeReader.create_sort_merge_reader(readers, None, None, spec, device=device)
    try:
        rd.execute()
        return rd.fetch()
    finally:
        rd.close()
