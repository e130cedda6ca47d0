"""Host-side mirror of the reference's file-format plugin SPI for the Parquet decode path.

  FileFormat / FileFormatFactory    paimon-common/src/main/java/org/apache/paimon/format/FileFormat.java:43-93,
                                    FileFormatFactory.java:28-32 (ServiceLoader lookup by identifier)
  FormatReaderFactory.createReader  paimon-common/.../format/FormatReaderFactory.java:33-57
  FormatReaderContext               paimon-common/.../format/FormatReaderContext.java:29-68
  ParquetFileFormat / ParquetReaderFactory   paimon-format/.../parquet/ParquetFileFormat.java:67-73,
                                    ParquetReaderFactory.java:113-148
  FileRecordReader.readBatch        paimon-common/.../reader/FileRecordReader.java

Same names and call order; the reader decodes the whole file on the device (libpaimon_gpu.so,
pg_parquet_*) and either hands the batch to the host (`read_batch`) or keeps it in HBM as the sorted run
of a merge (`as_sorted_run_reader`) — the fused decode -> merge path of KeyValueFileReaderFactory
(paimon-core/.../io/KeyValueFileReaderFactory.java:119-172).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import _native as N
from .columnar import KeyValueBatch
from .sort_merge_reader import RecordReader, SortedRunReader, _SchemaHandle, fetch_run
from .types import KeyValueSchema


class LocalFileIO:
    """Stand-in for org.apache.paimon.fs.FileIO: supplies the file's bytes (the Java side reads them with its
    own FileIO and passes a direct buffer)."""

    def read_bytes(self, path: str) -> bytes:
        with open(path, "rb") as f:
            return f.read()

    def get_file_size(self, path: str) -> int:
        import os
        return os.path.getsize(path)

    def write_bytes(self, path: str, data: bytes) -> None:
        with open(path, "wb") as f:
            f.write(data)


@dataclass
class FormatReaderContext:
    file_io: LocalFileIO
    file_path: str
    file_size: Optional[int] = None
    selection: Optional[object] = None      # RoaringBitmap32 row selection: refused (deletion vectors: dv_factory)


class FileRecordReader(RecordReader):
    pass


class ParquetFileRecordReader(FileRecordReader):
    """One KeyValue data file, decoded on the device."""

    def __init__(self, schema: KeyValueSchema, file_bytes: bytes, device: int = 0):
        self.schema = schema
        self.lib = N.init(device)
        self._schema_h = _SchemaHandle(schema, device)
        self._buf = np.frombuffer(file_bytes, dtype=np.uint8)
        h = C.c_uint64(0)
        try:
            N.check(self.lib.pg_parquet_open(self._schema_h.handle, self._buf.ctypes.data, len(self._buf), C.byref(h)))
        except Exception:
            self._schema_h.close()
            raise
        self._reader = h.value
        self._run = 0
        self._done = False

    def info(self) -> N.PgParquetInfo:
        info = N.PgParquetInfo()
        N.check(self.lib.pg_parquet_describe(self._reader, C.byref(info)))
        return info

    def _decode(self) -> int:
        if not self._run:
            h = C.c_uint64(0)
            N.check(self.lib.pg_parquet_read_run(self._reader, C.byref(h)))
            self._run = h.value
        return self._run

    def read_batch(self) -> Optional[KeyValueBatch]:
        """FileRecordReader.readBatch(): the whole file as one batch, then None (end of input)."""
        if self._done:
            return None
        self._done = True
        batch = fetch_run(self.schema, self._decode())
        return batch if batch.n_rows > 0 else None

    def as_sorted_run_reader(self) -> SortedRunReader:
        """Keep the decoded columns in HBM and hand them to a SortMergeReader (no host round trip).  The
        returned reader owns the run handle."""
        run = self._decode()
        self._run = 0
        return SortedRunReader.from_native_run(self.schema, self.info().n_rows, run)

    def close(self) -> None:
        lib = N.load()
        if self._run:
            lib.pg_run_free(self._run)
            self._run = 0
        if self._reader:
            lib.pg_parquet_free(self._reader)
            self._reader = 0
        if self._schema_h is not None:
            self._schema_h.close()
            self._schema_h = None


def read_section(schema: KeyValueSchema, files, n_runs: int, device: int = 0, check_names: bool = True,
                 read_value_fields=None, file_format: str = "parquet"):
    """Decode every data file of a section with ONE batch of device launches (pg_parquet_read_section, or
    pg_orc_read_section for file_format="orc") and return
    (one SortedRunReader per run, PgSectionInfo).  `files` = [(buffer, run index)], in key order inside a run; a
    buffer is bytes / a numpy uint8 array (host memory) or a (device pointer, size) tuple (bytes already in HBM).
    The files of a run are concatenated on the device, as MergeTreeReaders.readerForRun's ConcatRecordReader does
    (MergeTreeReaders.java:94-101): the merge gets k = number of runs inputs.  Columns are resolved by field name
    (missing nullable fields decode as NULL, extra file columns are ignored, INT -> BIGINT / FLOAT -> DOUBLE widen);
    `read_value_fields` (one bool per value field) is the read-type projection pushed into the decoder."""
    lib = N.init(device)
    sh = _SchemaHandle(schema, device)
    keep = []
    descs = (N.PgFileDesc * max(len(files), 1))()
    for i, (buf, run) in enumerate(files):
        if isinstance(buf, tuple):
            descs[i] = N.PgFileDesc(int(buf[0]), int(buf[1]), N.PG_MEM_DEVICE, int(run))
        else:
            arr = np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else np.ascontiguousarray(buf, np.uint8)
            keep.append(arr)
            descs[i] = N.PgFileDesc(arr.ctypes.data, len(arr), N.PG_MEM_HOST, int(run))
    names = None
    if check_names:
        nm = [f.name for f in schema.file_fields()]
        names = (C.c_char_p * len(nm))(*[x.encode() for x in nm])
    runs = (C.c_uint64 * max(n_runs, 1))()
    info = N.PgSectionInfo()
    mask = None
    if read_value_fields is not None:
        mask = np.array([1] * (schema.n_key + 2) + [1 if b else 0 for b in read_value_fields], np.uint8)
        keep.append(mask)
    try:
        fn = {"parquet": lib.pg_parquet_read_section, "orc": lib.pg_orc_read_section}.get(file_format.lower())
        if fn is None:
            raise N.UnsupportedOnDevice(2, f"file format '{file_format}' is not decoded on device (parquet and orc are)")
        N.check(fn(sh.handle, descs, len(files), n_runs, names, None if mask is None else mask.ctypes.data, runs,
                   C.byref(info)))
    finally:
        sh.close()
    readers = []
    for r in range(n_runs):
        n_rows = C.c_int64(0)
        N.check(lib.pg_run_layout(runs[r], C.byref(n_rows), None, None, schema.n_cols))
        readers.append(SortedRunReader.from_native_run(schema, int(n_rows.value), runs[r]))
    return readers, info


class FileUpload:
    """The data files of one section on their way to the device (pg_files_upload_begin): start it for section i + 1
    before decoding section i, and the host -> device copy of the encoded bytes — the longest leg of an end-to-end
    step — overlaps the decode, the merge and the read-back.  `files` = [(buffer, run index)] with page-locked host
    buffers (bytes / numpy uint8); wait() returns [((device pointer, size), run index)] for read_section()."""

    def __init__(self, files, device: int = 0):
        self._lib = N.init(device)
        self._keep = []
        self._runs = [int(r) for _, r in files]
        descs = (N.PgFileDesc * max(len(files), 1))()
        for i, (buf, run) in enumerate(files):
            if isinstance(buf, tuple):
                descs[i] = N.PgFileDesc(int(buf[0]), int(buf[1]), N.PG_MEM_DEVICE, int(run))
            else:
                arr = np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else np.ascontiguousarray(buf, np.uint8)
                self._keep.append(arr)
                descs[i] = N.PgFileDesc(arr.ctypes.data, len(arr), N.PG_MEM_HOST, int(run))
        h = C.c_uint64(0)
        N.check(self._lib.pg_files_upload_begin(descs, len(files), C.byref(h)))
        self._handle = h.value
        self._n = len(files)

    def wait(self):
        out = (N.PgFileDesc * max(self._n, 1))()
        N.check(self._lib.pg_files_upload_wait(self._handle, out, self._n))
        return [((int(out[i].bytes), int(out[i].size)), self._runs[i]) for i in range(self._n)]

    def close(self):
        if self._handle:
            N.check(self._lib.pg_files_upload_free(self._handle))
            self._handle = 0
            self._keep = []


class FormatReaderFactory:
    def create_reader(self, context: FormatReaderContext) -> FileRecordReader:
        raise NotImplementedError


class ParquetReaderFactory(FormatReaderFactory):
    def __init__(self, data_schema: KeyValueSchema, device: int = 0):
        self.data_schema = data_schema
        self.device = device

    def create_reader(self, context: FormatReaderContext) -> ParquetFileRecordReader:
        if context.selection is not None:
            raise N.UnsupportedOnDevice(2, "RoaringBitmap32 row selections are not pushed into the device decoder; deletion "
                                          "vectors are applied after the decode (KeyValueFileReaderFactory(dv_factory=...))")
        return ParquetFileRecordReader(self.data_schema, context.file_io.read_bytes(context.file_path), self.device)


class FileFormat:
    """FileFormat.fromIdentifier / createReaderFactory."""

    identifier = ""

    @staticmethod
    def from_identifier(identifier: str, device: int = 0) -> "FileFormat":
        if identifier.lower() == "parquet":
            return ParquetFileFormat(device)
        if identifier.lower() == "orc":
            return OrcFileFormat(device)
        raise N.UnsupportedOnDevice(2, f"file format '{identifier}' is not decoded on device (parquet and orc are; "
                                       f"avro data files stay on the Java side)")

    def create_reader_factory(self, data_schema: KeyValueSchema, projected=None, filters=None) -> FormatReaderFactory:
        raise NotImplementedError


class ParquetFileFormat(FileFormat):
    identifier = "parquet"

    def __init__(self, device: int = 0):
        self.device = device

    def create_reader_factory(self, data_schema: KeyValueSchema, projected=None, filters=None) -> ParquetReaderFactory:
        # keys are never projected before a merge and only key filters may be pushed into overlapping
        # sections (MergeFileSplitRead.java:204-213, 276-277): the merge path reads full files
        if projected is not None and projected != data_schema:
            raise N.UnsupportedOnDevice(2, "projection push-down is not applied on the merge path")
        return ParquetReaderFactory(data_schema, self.device)


class OrcFileRecordReader(FileRecordReader):
    """One ORC KeyValue data file, decoded on the device (pg_orc_read_section over a section of one file)."""

    def __init__(self, schema: KeyValueSchema, file_bytes: bytes, device: int = 0):
        self.schema = schema
        self.device = device
        self._bytes = file_bytes
        self._reader: Optional[SortedRunReader] = None
        self._info = None
        self._done = False

    def _decode(self) -> SortedRunReader:
        if self._reader is None:
            readers, self._info = read_section(self.schema, [(self._bytes, 0)], 1, self.device, file_format="orc")
            self._reader = readers[0]
        return self._reader

    def info(self):
        self._decode()
        return self._info

    def read_batch(self) -> Optional[KeyValueBatch]:
        if self._done:
            return None
        self._done = True
        batch = self._decode().read_batch()
        return batch if batch is not None and batch.n_rows > 0 else None

    def as_sorted_run_reader(self) -> SortedRunReader:
        r = self._decode()
        self._reader = None
        return r

    def close(self) -> None:
        if self._reader is not None:
            self._reader.close()
            self._reader = None


class OrcReaderFactory(FormatReaderFactory):
    """OrcReaderFactory.createReader (paimon-format/.../orc/OrcReaderFactory.java:98-163)."""

    def __init__(self, data_schema: KeyValueSchema, device: int = 0):
        self.data_schema = data_schema
        self.device = device

    def create_reader(self, context: FormatReaderContext) -> OrcFileRecordReader:
        if context.selection is not None:
            raise N.UnsupportedOnDevice(2, "RoaringBitmap32 row selections are not pushed into the device decoder")
        return OrcFileRecordReader(self.data_schema, context.file_io.read_bytes(context.file_path), self.device)


class OrcFileFormat(FileFormat):
    identifier = "orc"

    def __init__(self, device: int = 0):
        self.device = device

    def create_reader_factory(self, data_schema: KeyValueSchema, projected=None, filters=None) -> OrcReaderFactory:
        if projected is not None and projected != data_schema:
            raise N.UnsupportedOnDevice(2, "pass the read-type projection to MergeFileSplitRead.with_read_type")
        return OrcReaderFactory(data_schema, self.device)
