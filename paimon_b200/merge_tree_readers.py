"""Host orchestration of the merge path: files -> sections -> runs -> device merges -> one reader.

Mirrors (same names, same argument meaning):
  IntervalPartition.partition           paimon-core/.../mergetree/compact/IntervalPartition.java:67-125
  SortedRun                             paimon-core/.../mergetree/SortedRun.java:40-116
  MergeTreeReaders.readerForMergeTree / readerForSection / readerForRun
                                        paimon-core/.../mergetree/MergeTreeReaders.java:44-101
  ConcatRecordReader                    paimon-core/.../mergetree/compact/ConcatRecordReader.java:35-86
  MergeFileSplitRead.createMergeReader  paimon-core/.../operation/MergeFileSplitRead.java:269-316
  DataFileMeta (the fields the path needs)   paimon-core/.../io/DataFileMeta.java:66-89

The control flow stays on the host exactly where the reference has it (it only touches file *metadata*);
every section is merged by one SortMergeReader on the device, sections are key-disjoint so their outputs
concatenate.  Files of one run inside a section are key-disjoint and ordered, so a run is the concatenation of
its files (SortedRun.fromSorted): the device gets them as one run made of several decoded files.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence

import numpy as np

from . import _native as N
from .columnar import Column, KeyValueBatch
from .format import FileFormat, FormatReaderContext, LocalFileIO
from .merge_function import MergeFunctionFactory, MergeSpec
from .sort_merge_reader import RecordReader, SortedRunReader, SortMergeReader
from .types import KeyValueSchema, is_varlen


@dataclass
class DataFileMeta:
    """Input descriptor at the seam (DataFileMeta.java:66-89): what scan planning hands to the reader."""
    file_name: str
    file_size: int
    row_count: int
    min_key: object              # key bounds: an integer, a string / bytes, or a tuple of those (composite keys)
    max_key: object
    min_sequence_number: int = 0
    max_sequence_number: int = 0
    level: int = 0
    delete_row_count: int = 0
    embedded_index: Optional[bytes] = None     # the file index when it is small enough for the manifest
    extra_files: List[str] = field(default_factory=list)   # else its side file '<file_name>.index'


def comparable_key(k):
    """Key bound in the reference's comparison order: strings compare as their UTF-8 bytes
    (BinaryString.java:109-126), tuples field by field."""
    if isinstance(k, str):
        return k.encode("utf-8")
    if isinstance(k, tuple):
        return tuple(comparable_key(x) for x in k)
    return k


@dataclass
class SortedRun:
    files: List[DataFileMeta] = field(default_factory=list)

    @staticmethod
    def from_sorted(files: Sequence[DataFileMeta]) -> "SortedRun":
        run = SortedRun(list(files))
        run.validate()
        return run

    def validate(self) -> None:                       # SortedRun.java:85-95
        for a, b in zip(self.files, self.files[1:]):
            if not comparable_key(a.max_key) < comparable_key(b.min_key):
                raise ValueError("SortedRun is not sorted and may contain overlapping key intervals")

    def total_size(self) -> int:
        return sum(f.file_size for f in self.files)


class IntervalPartition:
    """Sections (key-disjoint) of runs (fewest non-overlapping file chains).  The algorithm runs in
    libpaimon_gpu.so's host code (pg_interval_partition) so that Java and Python share one implementation."""

    def __init__(self, input_files: Sequence[DataFileMeta]):
        self.files = list(input_files)

    def partition(self) -> List[List[SortedRun]]:
        n = len(self.files)
        if n == 0:
            return []
        lib = N.load()
        lo = [comparable_key(f.min_key) for f in self.files]
        hi = [comparable_key(f.max_key) for f in self.files]
        if all(isinstance(k, (int, np.integer)) for k in lo + hi):
            mn, mx = np.array(lo, np.int64), np.array(hi, np.int64)
        else:
            # the algorithm only compares key bounds: dense ranks of the bounds give the same sections and runs
            rank = {k: i for i, k in enumerate(sorted(set(lo + hi)))}
            mn = np.array([rank[k] for k in lo], np.int64)
            mx = np.array([rank[k] for k in hi], np.int64)
        sec = np.zeros(n, np.int32)
        run = np.zeros(n, np.int32)
        ns = C.c_int32(0)
        N.check(lib.pg_interval_partition(n, mn.ctypes.data, mx.ctypes.data, sec.ctypes.data, run.ctypes.data,
                                          C.byref(ns)))
        sections: List[dict] = [dict() for _ in range(ns.value)]
        for i, f in enumerate(self.files):
            sections[sec[i]].setdefault(int(run[i]), []).append(f)
        out = []
        for s in sections:
            runs = []
            for rid in sorted(s):
                files = sorted(s[rid], key=lambda f: (comparable_key(f.min_key), comparable_key(f.max_key)))
                runs.append(SortedRun.from_sorted(files))
            out.append(runs)
        return out


class ConcatRecordReader(RecordReader):
    """Readers are opened lazily one after the other (ConcatRecordReader.java:52-75)."""

    def __init__(self, suppliers: Sequence[Callable[[], RecordReader]]):
        self.queue = list(suppliers)
        self.current: Optional[RecordReader] = None

    def read_batch(self) -> Optional[KeyValueBatch]:
        while True:
            if self.current is not None:
                batch = self.current.read_batch()
                if batch is not None:
                    return batch
                self.current.close()
                self.current = None
            if not self.queue:
                return None
            self.current = self.queue.pop(0)()

    def close(self) -> None:
        if self.current is not None:
            self.current.close()
            self.current = None


def concat_batches(schema: KeyValueSchema, batches: Sequence[KeyValueBatch]) -> KeyValueBatch:
    """Concatenate key-disjoint, ordered batches (host helper for tests / small results)."""
    if not batches:
        return KeyValueBatch.from_rows(schema, [])
    cols = []
    for ci, t in enumerate(schema.physical_types()):
        parts = [b.columns[ci].canonical() for b in batches]
        from .columnar import pack_validity, unpack_validity
        valid = np.concatenate([unpack_validity(p.valid, len(p)) for p in parts])
        if is_varlen(t):
            data = np.concatenate([p.data for p in parts]) if parts else np.zeros(0, np.uint8)
            offs = [np.zeros(1, np.int64)]
            base = 0
            for p in parts:
                offs.append(p.offsets[1:].astype(np.int64) + base)
                base += int(p.offsets[-1])
            cols.append(Column(t, data, np.concatenate(offs).astype(np.int32), pack_validity(valid)))
        else:
            cols.append(Column(t, np.concatenate([p.data for p in parts]), None, pack_validity(valid)))
    return KeyValueBatch(schema, cols)


class KeyValueFileReaderFactory:
    """createRecordReader(file) — KeyValueFileReaderFactory.java:119-172: format by file suffix, decode on the
    device.  (Schema evolution mappings and deletion vectors are applied on the Java side today.)"""

    def __init__(self, schema: KeyValueSchema, file_io: Optional[LocalFileIO] = None, device: int = 0,
                 dv_factory: Optional[Callable[[str], Optional[Sequence[int]]]] = None):
        self.schema = schema
        self.file_io = file_io or LocalFileIO()
        self.device = device
        # DeletionVector.Factory (KeyValueFileReaderFactory.java:119-172 wraps the reader in
        # ApplyDeletionVectorReader when the file has a deletion vector): file name -> deleted row positions
        self.dv_factory = dv_factory

    def create_record_reader(self, meta: DataFileMeta):
        suffix = meta.file_name.rsplit(".", 1)[-1]
        fmt = FileFormat.from_identifier(suffix, self.device)
        return fmt.create_reader_factory(self.schema).create_reader(
            FormatReaderContext(self.file_io, meta.file_name, meta.file_size))


class MergeTreeReaders:
    @staticmethod
    def _read_files(metas: Sequence[DataFileMeta], reader_factory: KeyValueFileReaderFactory) -> List[bytes]:
        """FileIO reads of the section's files (concurrent: the device decode starts once all bytes are there)."""
        for m in metas:                                   # format by file-name suffix (KeyValueFileReaderFactory.java:119-172)
            FileFormat.from_identifier(m.file_name.rsplit(".", 1)[-1], reader_factory.device)
        if len(metas) <= 1:
            return [reader_factory.file_io.read_bytes(m.file_name) for m in metas]
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=min(8, len(metas))) as ex:
            return list(ex.map(lambda m: reader_factory.file_io.read_bytes(m.file_name), metas))

    @staticmethod
    def open_runs(section: Sequence[SortedRun], reader_factory: KeyValueFileReaderFactory,
                  read_value_fields=None) -> List[SortedRunReader]:
        """The sorted runs of a section as device-resident merge inputs: ONE batch of decode launches for all files
        (pg_parquet_read_section), and a run = the concatenation of its key-disjoint files, like readerForRun's
        ConcatRecordReader (MergeTreeReaders.java:94-101) — so the merge fan-in is the number of RUNS, not files.
        Deletion vectors (ApplyDeletionVectorReader) are applied per run with the files' positions shifted by the
        file's row offset inside the run."""
        from .format import read_section
        metas, run_of = [], []
        for r, run in enumerate(section):
            for m in run.files:
                metas.append(m)
                run_of.append(r)
        blobs = MergeTreeReaders._read_files(metas, reader_factory)
        formats = {m.file_name.rsplit(".", 1)[-1].lower() for m in metas} or {"parquet"}
        if len(formats) > 1:
            raise N.UnsupportedOnDevice(2, f"a section mixes file formats {sorted(formats)}: decoded per format on the Java side")
        readers, _ = read_section(reader_factory.schema, list(zip(blobs, run_of)), len(section), reader_factory.device,
                                  read_value_fields=read_value_fields, file_format=formats.pop())
        if reader_factory.dv_factory is not None:
            from .sort_merge_reader import apply_deletion_vector
            row0 = [0] * len(section)
            deleted: List[List[int]] = [[] for _ in section]
            for m, r in zip(metas, run_of):
                d = reader_factory.dv_factory(m.file_name)
                if d is not None and len(d):
                    deleted[r] += [int(p) + row0[r] for p in d if 0 <= int(p) < m.row_count]
                row0[r] += m.row_count
            for r, d in enumerate(deleted):
                if d:
                    filtered = apply_deletion_vector(reader_factory.schema, readers[r], d, device=reader_factory.device)
                    readers[r].close()
                    readers[r] = filtered
        return readers

    @staticmethod
    def reader_for_run(run: SortedRun, reader_factory: KeyValueFileReaderFactory) -> SortedRunReader:
        """MergeTreeReaders.readerForRun (:94-101): the run's files, concatenated, as one merge input."""
        return MergeTreeReaders.open_runs([run], reader_factory)[0]

    @staticmethod
    def reader_for_section(section: Sequence[SortedRun], reader_factory: KeyValueFileReaderFactory,
                           user_defined_seq_comparator, merge_function_wrapper: MergeSpec) -> RecordReader:
        """MergeTreeReaders.readerForSection (:67-92).  One device merge takes at most PG_MAX_RUNS = 32 sorted runs;
        a section with more runs (the reference's MergeSorter, MergeSorter.java:112-198, spills the smallest ones and
        still merges all of them at once) is merged in rounds when the merge function allows it exactly."""
        spec_n = merge_function_wrapper.normalised(reader_factory.schema.n_val)
        if user_defined_seq_comparator is not None and hasattr(user_defined_seq_comparator, "apply"):
            spec_n = user_defined_seq_comparator.apply(spec_n)
        decode_mask = spec_n.fields_the_merge_reads(reader_factory.schema.n_val) if spec_n.read_fields else None
        runs = MergeTreeReaders.open_runs(section, reader_factory, read_value_fields=decode_mask)
        inner: List[SortMergeReader] = []
        try:
            if len(runs) > 32:
                runs = MergeTreeReaders._merge_in_rounds(runs, user_defined_seq_comparator, merge_function_wrapper,
                                                         reader_factory, inner)
            merge = SortMergeReader.create_sort_merge_reader(runs, None, user_defined_seq_comparator,
                                                             merge_function_wrapper, device=reader_factory.device)
        except Exception:
            for r in runs:
                r.close()
            for m in inner:
                m.close()
            raise

        class _Section(RecordReader):
            def read_batch(self_inner):
                return merge.read_batch()

            def close(self_inner):
                merge.close()                            # closes its run readers too
                for m in inner:
                    m.close()
        return _Section()

    @staticmethod
    def _merge_in_rounds(runs: List[SortedRunReader], udsc, spec: MergeSpec, reader_factory, inner: list):
        """More than 32 sorted runs: groups of 32 are merged into intermediate runs (views of the group merges'
        device batches, no copy), until at most 32 remain for the final merge.  Pre-reducing a group is exact only
        when the merge function's result is one of the group's input records, chosen by an order that does not
        depend on the other groups: deduplicate (the newest record, retracts skipped under 'ignore-delete') and
        first-row.  partial-update and aggregation fold every record of a key in global sequence order (a column of
        group A's result may be older than group B's value for it; floating-point sums are not associative), so
        they are refused instead of being merged approximately."""
        from .merge_function import MergeEngine
        if spec.engine not in (MergeEngine.DEDUPLICATE, MergeEngine.FIRST_ROW) or spec.read_fields:
            for r in runs:
                r.close()
            raise N.UnsupportedOnDevice(2, "more than 32 sorted runs in one section are merged in rounds for the "
                                           "deduplicate and first-row merge engines only (without a read-type "
                                           "projection); partial-update / aggregation need one pass over all runs")
        lib = N.load()
        step = spec.with_drop_delete(False)              # deletes must survive until the last round
        while len(runs) > 32:
            nxt: List[SortedRunReader] = []
            for g in range(0, len(runs), 32):
                group = runs[g:g + 32]
                if len(group) == 1:
                    nxt.append(group[0])
                    continue
                m = SortMergeReader.create_sort_merge_reader(group, None, udsc, step, device=reader_factory.device)
                inner.append(m)                          # owns the group's runs and the intermediate batch
                m.execute()
                n_out = m.device_batch().n_rows
                h, start = C.c_uint64(0), C.c_int64(0)
                N.check(lib.pg_run_slice(m._merge_h, 0, n_out, C.byref(h), C.byref(start)))
                nxt.append(SortedRunReader.from_native_run(reader_factory.schema, n_out, h.value))
            runs = nxt
        return runs

    @staticmethod
    def reader_for_merge_tree(sections: Sequence[Sequence[SortedRun]], reader_factory: KeyValueFileReaderFactory,
                              user_defined_seq_comparator, merge_function_wrapper: MergeSpec) -> RecordReader:
        """MergeTreeReaders.readerForMergeTree (:44-65): ConcatRecordReader over lazily opened section readers."""
        return ConcatRecordReader([
            (lambda s=s: MergeTreeReaders.reader_for_section(s, reader_factory, user_defined_seq_comparator,
                                                             merge_function_wrapper))
            for s in sections])


class MergeFileSplitRead:
    """createMergeReader(partition, bucket, files, deletionVectors, keepDelete) — MergeFileSplitRead.java:269-316:
    sections from IntervalPartition, one merge per section, DropDeleteReader unless forceKeepDelete."""

    def __init__(self, schema: KeyValueSchema, mf_factory: MergeFunctionFactory, user_defined_seq_comparator=None,
                 file_io: Optional[LocalFileIO] = None, device: int = 0):
        self.schema = schema
        self.mf_factory = mf_factory
        self.udsc = user_defined_seq_comparator
        self.reader_factory = KeyValueFileReaderFactory(schema, file_io, device)
        self.force_keep_delete = False

    def force_keep_delete_(self) -> "MergeFileSplitRead":      # forceKeepDelete()
        self.force_keep_delete = True
        return self

    def with_read_type(self, field_names: Sequence[str]) -> "MergeFileSplitRead":
        """withReadType (MergeFileSplitRead.java:133-163): the value fields the engine wants.  The projection is pushed
        into the decoder (column chunks of other fields are not decoded) and into the merge (no output columns, no emit
        work for them); keys are never projected before the merge (:276-277), and fields the merge function compares
        ('sequence.field', sequence groups) are still decoded (adjustReadType)."""
        names = self.schema.value_type.field_names()
        unknown = [n for n in field_names if n not in names]
        if unknown:
            raise ValueError(f"read type has fields the table does not have: {unknown}")
        wanted = set(field_names)
        self.read_fields = [n in wanted for n in names]
        return self

    def with_key_filter(self, lower=None, upper=None) -> "MergeFileSplitRead":
        """withFilter (MergeFileSplitRead.java:181-217): only KEY predicates may be pushed below the merge — a value
        predicate would drop the newer version of a row and resurrect an older one (comment :204-213).  Here the
        key predicate is a closed range on the primary key; it prunes data files by their key bounds before
        IntervalPartition (a file without keys in range cannot contribute to any key in range).  Rows outside
        the range that live in surviving files are still returned: the engine filters above the reader, as in
        the reference."""
        self.key_lower, self.key_upper = lower, upper
        return self

    def _prune(self, files: Sequence[DataFileMeta]) -> List[DataFileMeta]:
        lo, hi = getattr(self, "key_lower", None), getattr(self, "key_upper", None)
        lo = None if lo is None else comparable_key(lo)
        hi = None if hi is None else comparable_key(hi)
        return [f for f in files if not ((lo is not None and comparable_key(f.max_key) < lo) or
                                         (hi is not None and comparable_key(f.min_key) > hi))]

    def create_merge_reader(self, files: Sequence[DataFileMeta], keep_delete: Optional[bool] = None) -> RecordReader:
        keep = self.force_keep_delete if keep_delete is None else keep_delete
        spec = self.mf_factory.create().with_drop_delete(not keep)      # DropDeleteReader fused into the merge
        if getattr(self, "read_fields", None) is not None:
            spec = spec.with_read_fields(self.read_fields)
        sections = IntervalPartition(self._prune(files)).partition()
        return MergeTreeReaders.reader_for_merge_tree(sections, self.reader_factory, self.udsc, spec)
