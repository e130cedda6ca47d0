"""The rewrite side of a compaction: merged device batch -> Parquet or ORC data files + DataFileMeta.

Mirrors (same names, same argument meaning):
  KeyValueDataFileWriter.write / result      paimon-core/.../io/KeyValueDataFileWriter.java:108-184
  RollingFileWriterImpl                      paimon-core/.../io/RollingFileWriterImpl.java:64-105
  MergeTreeCompactRewriter.rewriteCompaction paimon-core/.../mergetree/compact/MergeTreeCompactRewriter.java:78-116
  CompactResult(before, after)               paimon-core/.../compact/CompactResult.java

The merge of a section, the drop-delete filter, the Parquet or ORC encode and the file statistics all happen on the
device; the host writes the encoded bytes through the FileIO and assembles the DataFileMeta.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _native as N
from .file_index import DataFileIndexWriter, FileIndexOptions
from .format import LocalFileIO
from .merge_function import MergeFunctionFactory
from .merge_tree_readers import (DataFileMeta, IntervalPartition, KeyValueFileReaderFactory, MergeTreeReaders,
                                 SortedRun)
from .sort_merge_reader import SortMergeReader
from .types import KeyValueSchema, PhysicalType, is_varlen, orc_column_type


@dataclass
class SimpleColStats:
    """min / max / nullCount of one column (SimpleColStats in paimon-common/.../format/SimpleColStats.java)."""
    min: object
    max: object
    null_count: int


@dataclass
class WrittenFile:
    meta: DataFileMeta
    value_stats: List[SimpleColStats]
    ms_encode: float
    n_pages: int


# Parquet CompressionCodec numbers (parquet.thrift) by the names Paimon's options use
PARQUET_CODECS = {"none": 0, "uncompressed": 0, "snappy": 1, "gzip": 2, "lzo": 3, "brotli": 4, "lz4": 5, "zstd": 6,
                  "lz4_raw": 7}


# ORC CompressionKind numbers (orc_proto) by the names 'orc.compress' and 'file.compression' use
ORC_CODECS = {"none": 0, "uncompressed": 0, "zlib": 1, "snappy": 2, "lzo": 3, "lz4": 4, "zstd": 5, "brotli": 6}

FILE_FORMATS = ("parquet", "orc")


def _per_level(value) -> Dict[int, str]:
    """'file.compression.per.level' / 'file.format.per.level' as a map: a dict, or the option's string form
    '0:lz4,5:zstd'."""
    if isinstance(value, dict):
        return {int(k): str(v) for k, v in value.items()}
    out = {}
    for item in str(value).split(","):
        if item.strip():
            k, v = item.split(":", 1)
            out[int(k.strip())] = v.strip()
    return out


def compression_for_level(options: Optional[Dict[str, object]], level: int) -> Tuple[str, int]:
    """(codec name, zstd level) of a data file written at `level`, the way the reference chooses them:
    'file.compression.per.level' for the level, else 'file.compression' (default zstd) (KeyValueFileWriterFactory.java
    :312-321, CoreOptions.java:299-323), overridden by 'parquet.compression' (RowDataParquetBuilder.java:121-122); the
    level is 'parquet.compression.codec.zstd.level', else 'file.compression.zstd-level' (default 1;
    ParquetFileFormat.java:98-101, CoreOptions.java:325-330)."""
    options = options or {}
    per_level = _per_level(options.get("file.compression.per.level", {}))
    codec = per_level.get(level, options.get("file.compression", "zstd"))
    codec = str(options.get("parquet.compression", codec)).lower()
    zstd_level = int(options.get("parquet.compression.codec.zstd.level", options.get("file.compression.zstd-level", 1)))
    return codec, zstd_level


def format_for_level(options: Optional[Dict[str, object]], level: int) -> str:
    """The file format of a data file written at `level`: 'file.format.per.level' for the level, else 'file.format',
    else parquet (KeyValueFileWriterFactory.java:301-310, CoreOptions.java:292-313)."""
    options = options or {}
    per_level = _per_level(options.get("file.format.per.level", {}))
    return str(per_level.get(level, options.get("file.format", "parquet"))).lower()


def orc_compression_for_level(options: Optional[Dict[str, object]], level: int) -> Tuple[str, int, int]:
    """(codec name, zstd level, compression block size) of an ORC data file written at `level`: the codec is
    'file.compression.per.level' for the level, else 'file.compression' (default zstd), overridden by 'orc.compress'
    (OrcWriterFactory.java:101-104); the level is 'orc.compression.zstd.level', else 'file.compression.zstd-level'
    (default 1; OrcFileFormat.java:158-175); the block size is 'orc.compress.size' (0 = the library's 256 KiB)."""
    options = options or {}
    per_level = _per_level(options.get("file.compression.per.level", {}))
    codec = per_level.get(level, options.get("file.compression", "zstd"))
    codec = str(options.get("orc.compress", codec)).lower()
    zstd_level = int(options.get("orc.compression.zstd.level", options.get("file.compression.zstd-level", 1)))
    return codec, zstd_level, int(options.get("orc.compress.size", 0))


# orc-core's smallest row index stride (WriterImpl.MIN_ROW_INDEX_STRIDE), and the largest bloom filter the device
# builds: the shared memory of one CTA (kBloomMaxBytes in orc_encode.cu)
ORC_MIN_ROW_INDEX_STRIDE = 1000
ORC_BLOOM_MAX_BYTES = 227 << 10


def orc_bloom_bits(entries: int, fpp: float) -> int:
    """The bits of an ORC bloom filter for `entries` values at `fpp`, as orc-core's BloomFilter sizes it."""
    nb = int(-entries * math.log(fpp) / (math.log(2) ** 2))
    return nb + 64 - nb % 64


def orc_index_options(schema: KeyValueSchema, stride: int, bloom_columns: Sequence[str], fpp: float):
    """pg_orc_index_options for a row index of `stride` rows per row group and bloom filters of the value fields
    `bloom_columns`.  The refusals of pg_orc_encode_indexed are raised here, before any device work."""
    stride, bloom_columns = int(stride), list(bloom_columns)
    invalid = None
    if stride < 0 or 0 < stride < ORC_MIN_ROW_INDEX_STRIDE:
        invalid = f"row index stride {stride} is negative or below {ORC_MIN_ROW_INDEX_STRIDE}"
    elif bloom_columns and stride == 0:
        invalid = "bloom filters need a row index stride"
    elif bloom_columns and not 0 < fpp < 1:
        invalid = f"bloom filter fpp {fpp} outside (0, 1)"
    elif len(set(bloom_columns)) != len(bloom_columns):
        invalid = f"bloom filter columns {bloom_columns} list a column twice"
    if invalid:
        raise N.PaimonGpuError(1, f"orc encode: {invalid}")
    if stride % 8:
        raise N.UnsupportedOnDevice(2, f"orc encode: row index stride {stride} is not a multiple of 8")
    by_name = {f.name: i for i, f in enumerate(schema.value_type.fields)}
    cols = []
    for name in bloom_columns:
        if name not in by_name:
            raise N.PaimonGpuError(1, f"orc encode: bloom filter column {name!r} is not a value field")
        t = schema.value_type.fields[by_name[name]].type
        if orc_column_type(t)[0] in (0, 14):                               # BOOLEAN, DECIMAL
            raise N.UnsupportedOnDevice(2, f"orc encode: bloom filter column {name!r} is {t}")
        cols.append(schema.n_key + 2 + by_name[name])
    if cols and orc_bloom_bits(stride, fpp) // 8 > ORC_BLOOM_MAX_BYTES:
        raise N.UnsupportedOnDevice(2, f"orc encode: a bloom filter of {stride} rows at fpp {fpp} is larger than "
                                       f"{ORC_BLOOM_MAX_BYTES} bytes")
    arr = (C.c_int32 * max(len(cols), 1))(*cols)
    opts = N.PgOrcIndexOptions(stride, len(cols), arr, float(fpp))
    opts._keep = arr
    return opts


def orc_index_for_level(options: Optional[Dict[str, object]]) -> Dict[str, object]:
    """The row index arguments of KeyValueDataFileWriter for an ORC output level, from the table options as orc-core
    reads them: 'orc.create.index' (default true), 'orc.row.index.stride' (default 10000), 'orc.bloom.filter.columns'
    (comma-separated, no default) and 'orc.bloom.filter.fpp' (default 0.01) (OrcConf.java:57-67,140-201).  Without an
    index there are no bloom filters either."""
    options = options or {}
    if str(options.get("orc.create.index", "true")).lower() != "true":
        return dict(row_index_stride=0, bloom_filter_columns=())
    cols = [c.strip() for c in str(options.get("orc.bloom.filter.columns", "")).split(",") if c.strip()]
    return dict(row_index_stride=int(options.get("orc.row.index.stride", 10000)), bloom_filter_columns=tuple(cols),
                bloom_filter_fpp=float(options.get("orc.bloom.filter.fpp", 0.01)))


def file_column_names(schema: KeyValueSchema) -> List[str]:
    """[_KEY_*, _SEQUENCE_NUMBER, _VALUE_KIND, value...] (KeyValue.schema, KeyValue.java:130-138)."""
    return [f.name for f in schema.file_fields()]


# parquet-mr's bloom filter fpp when 'parquet.bloom.filter.fpp#<col>' is not set (ParquetProperties)
PARQUET_BLOOM_DEFAULT_FPP = 0.01


def parquet_bloom_for_level(schema: KeyValueSchema, options: Optional[Dict[str, object]]) -> List[Tuple[int, int, float]]:
    """The Parquet bloom filters of a data file as (file column, ndv, fpp), from the table options parquet-mr receives
    (RowDataParquetBuilder.java:96-116; options starting with 'parquet.' keep the prefix, FileFormat
    .getIdentifierPrefixOptions).  'parquet.bloom.filter.enabled' (default false) covers every file column, _KEY_<pk>,
    _SEQUENCE_NUMBER and _VALUE_KIND included, and 'parquet.bloom.filter.enabled#<col>' overrides it for one column
    either way; 'parquet.bloom.filter.expected.ndv#<col>' (0 = unset: a 1 MiB filter) and
    'parquet.bloom.filter.fpp#<col>' (default 0.01) size its filter.  A '#<col>' naming no file column is ignored, as
    ColumnConfigParser ignores it.  BOOLEAN columns get no filter: the Parquet specification defines no BOOLEAN hash.
    A malformed ndv or fpp, or one outside ndv > 0 / 0 < fpp < 1, is refused here, before any device work."""
    options = options or {}
    ndv, fpp = {}, {}
    for key, value in options.items():
        for prefix, out, parse in (("parquet.bloom.filter.expected.ndv#", ndv, int),
                                   ("parquet.bloom.filter.fpp#", fpp, float)):
            if not str(key).startswith(prefix):
                continue
            try:
                v = parse(str(value).strip())
            except ValueError:
                raise N.PaimonGpuError(1, f"parquet encode: option {key} = {value!r} is not a number") from None
            if not (v > 0 if parse is int else 0 < v < 1):
                raise N.PaimonGpuError(1, f"parquet encode: option {key} = {value!r} is outside "
                                          f"{'ndv > 0' if parse is int else '(0, 1)'}")
            out[str(key)[len(prefix):]] = v
    enabled = str(options.get("parquet.bloom.filter.enabled", "false")).strip().lower() == "true"
    out = []
    for c, (name, t) in enumerate(zip(file_column_names(schema), schema.physical_types())):
        on = options.get(f"parquet.bloom.filter.enabled#{name}")
        if (enabled if on is None else str(on).strip().lower() == "true") and t != PhysicalType.BOOL:
            out.append((c, ndv.get(name, 0), fpp.get(name, PARQUET_BLOOM_DEFAULT_FPP)))
    return out


class KeyValueDataFileWriter:
    """Encodes rows [row0, row0 + n_rows) of a device batch (a merge handle holding a batch, or a run handle) as
    one data file of `file_format` ('parquet' or 'orc') and returns its DataFileMeta.  `compression` names the codec
    ('none' or 'zstd', compressed on the device; the library refuses the others), `zstd_level` is
    file.compression.zstd-level.  Parquet takes `row_group_rows` / `page_rows`, ORC `stripe_rows` /
    `compression_block_size` and writes the logical types of the schema (OrcTypeUtil.convertToOrcType).  With
    `file_index` (the table's 'file-index.*' options) the file gets the bloom filters of its value columns, built on
    the device over the rows of the file, as DataFileMeta.embedded_index or the side file of extra_files
    (KeyValueDataFileWriter.java:103-113,156-181); options the device cannot build are refused here, before any
    device work.  With `page_index` a Parquet file carries the ColumnIndex and OffsetIndex of every column chunk
    (the page bounds computed on the device), as parquet-mr writes them; ORC files ignore it.  An ORC file takes
    `row_index_stride` (rows per row group of its row index, 0 = none), `bloom_filter_columns` (value-field names
    with a bloom filter per row group, built on the device) and `bloom_filter_fpp`, as orc-core writes them for
    'orc.row.index.stride', 'orc.bloom.filter.columns' and 'orc.bloom.filter.fpp'; Parquet files ignore them.  Index
    options the device cannot write are refused here, before any device work.  A Parquet file takes `parquet_bloom`,
    (file column, ndv, fpp) per column with a Parquet bloom filter per row group (parquet_bloom_for_level), built on the
    device; ORC files ignore it."""

    def __init__(self, schema: KeyValueSchema, path: str, level: int, file_io: Optional[LocalFileIO] = None,
                 row_group_rows: int = 0, page_rows: int = 0, compression: str = "none", zstd_level: int = 1,
                 file_format: str = "parquet", stripe_rows: int = 0, compression_block_size: int = 0,
                 file_index: Optional[FileIndexOptions] = None, page_index: bool = False,
                 row_index_stride: int = 0, bloom_filter_columns: Sequence[str] = (), bloom_filter_fpp: float = 0.01,
                 parquet_bloom: Sequence[Tuple[int, int, float]] = ()):
        self.schema = schema
        self.path = path
        self.level = level
        self.file_io = file_io or LocalFileIO()
        self.file_format = file_format.lower()
        if self.file_format not in FILE_FORMATS:
            raise N.UnsupportedOnDevice(2, f"file format '{file_format}' is not written on the device (parquet and orc are)")
        codecs = ORC_CODECS if self.file_format == "orc" else PARQUET_CODECS
        if compression.lower() not in codecs:
            raise ValueError(f"unknown {self.file_format} file compression {compression!r}")
        self.codec = codecs[compression.lower()]
        self.zstd_level = int(zstd_level)
        self.opts = N.PgParquetWriteOptions(row_group_rows, page_rows, int(bool(page_index)))
        if self.file_format == "orc":
            fields = schema.file_fields()
            self._orc_types = (N.PgOrcColumnType * len(fields))(*[N.PgOrcColumnType(*orc_column_type(f.type))
                                                                   for f in fields])
            self.orc_opts = N.PgOrcWriteOptions(stripe_rows, self.codec, self.zstd_level, compression_block_size,
                                                self._orc_types)
            self.orc_index = orc_index_options(schema, row_index_stride, bloom_filter_columns, bloom_filter_fpp)
        bloom = list(parquet_bloom)
        self._bloom_cols = (N.PgParquetBloomColumn * max(len(bloom), 1))(
            *[N.PgParquetBloomColumn(int(c), int(ndv), float(fpp)) for c, ndv, fpp in bloom])
        self.parquet_bloom = N.PgParquetBloomOptions(len(bloom), self._bloom_cols)
        self.index_writer = None
        if file_index is not None and not file_index.is_empty():
            self.index_writer = DataFileIndexWriter(schema, file_index)
        self.lib = N.load()

    def write(self, source_handle: int, row0: int = 0, n_rows: int = -1) -> WrittenFile:
        names = file_column_names(self.schema)
        arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
        fh = C.c_uint64(0)
        if self.file_format == "orc":
            N.check(self.lib.pg_orc_encode_indexed(source_handle, arr, row0, n_rows, C.byref(self.orc_opts),
                                                   C.byref(self.orc_index), C.byref(fh)))
        else:
            N.check(self.lib.pg_parquet_encode_bloom(source_handle, arr, row0, n_rows, C.byref(self.opts), self.codec,
                                                     self.zstd_level, C.byref(self.parquet_bloom), C.byref(fh)))
        try:
            meta = N.PgFileMeta()
            N.check(self.lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
            buf = np.empty(max(meta.file_bytes, 1), np.uint8)
            N.check(self.lib.pg_parquet_file_fetch(fh.value, buf.ctypes.data, meta.file_bytes))
            with open(self.path, "wb") as f:
                f.write(buf[: meta.file_bytes].tobytes())
            stats = [self._column_stats(fh.value, c) for c in range(self.schema.n_cols)]
        finally:
            self.lib.pg_parquet_file_free(fh.value)
        # min / max key = the key ROW of the first / last record of the file (the batch is sorted by key):
        # KeyValueDataFileWriter.java:116-118,166-167 keeps the first and the last key it saw.  Every key field,
        # var-len ones included — column statistics would truncate composite keys and have nothing for strings.
        n_file = int(meta.n_rows)
        min_key = max_key = None
        if n_file > 0:
            min_key = self._key_row(source_handle, row0)
            max_key = self._key_row(source_handle, row0 + n_file - 1)
        dfm = DataFileMeta(file_name=self.path, file_size=int(meta.file_bytes), row_count=n_file,
                           min_key=min_key, max_key=max_key,
                           min_sequence_number=int(meta.min_sequence_number),
                           max_sequence_number=int(meta.max_sequence_number), level=self.level,
                           delete_row_count=int(meta.delete_row_count))
        if self.index_writer is not None:
            index = self.index_writer.write(self.file_io, self.path, source_handle, row0, n_file)
            dfm.embedded_index, dfm.extra_files = index.embedded_index, index.extra_files
        return WrittenFile(dfm, stats[self.schema.n_key + 2:], float(meta.ms_encode), int(meta.n_pages))

    def _key_row(self, source_handle: int, row: int):
        """The primary key of one row of the device batch: a scalar for single-field keys, else a tuple."""
        from .sort_merge_reader import fetch_slice
        one = fetch_slice(self.schema, source_handle, row, row + 1)
        vals = [one.columns[i].to_pylist()[0] for i in range(self.schema.n_key)]
        return vals[0] if len(vals) == 1 else tuple(vals)

    def _column_stats(self, fh: int, c: int) -> SimpleColStats:
        nulls, has = C.c_int64(0), C.c_int32(0)
        mn, mx = np.zeros(1, np.int64), np.zeros(1, np.int64)
        N.check(self.lib.pg_parquet_file_column_stats(fh, c, C.byref(nulls), C.byref(has), mn.ctypes.data,
                                                      mx.ctypes.data))
        if not has.value:
            return SimpleColStats(None, None, int(nulls.value))
        t = self.schema.physical_types()[c]
        if t in (PhysicalType.FLOAT, PhysicalType.DOUBLE):
            return SimpleColStats(float(mn.view(np.float64)[0]), float(mx.view(np.float64)[0]), int(nulls.value))
        if t == PhysicalType.BOOL:
            return SimpleColStats(bool(mn[0]), bool(mx[0]), int(nulls.value))
        return SimpleColStats(int(mn[0]), int(mx[0]), int(nulls.value))


class RollingFileWriter:
    """Cuts one batch into files of at most `target_file_rows` rows (the reference rolls on the byte size of the
    output stream, RollingFileWriterImpl.java:85-100; rows are what the device knows before encoding).  Every file
    takes `writer_args` (KeyValueDataFileWriter's arguments) and `page_index`."""

    def __init__(self, schema: KeyValueSchema, directory: str, level: int, target_file_rows: int,
                 file_io: Optional[LocalFileIO] = None, prefix: str = "data", page_index: bool = False,
                 **writer_args):
        self.schema, self.directory, self.level = schema, directory, level
        self.target = max(8, (int(target_file_rows) + 7) & ~7)       # files start at multiples of 8 rows
        self.file_io = file_io
        self.prefix = prefix
        self.writer_args = dict(writer_args, page_index=page_index)
        self.suffix = writer_args.get("file_format", "parquet").lower()
        self.results: List[WrittenFile] = []

    def write(self, source_handle: int, n_rows: int) -> List[WrittenFile]:
        for i, r0 in enumerate(range(0, n_rows, self.target)):
            path = os.path.join(self.directory, f"{self.prefix}-{len(self.results)}.{self.suffix}")
            w = KeyValueDataFileWriter(self.schema, path, self.level, self.file_io, **self.writer_args)
            self.results.append(w.write(source_handle, r0, min(self.target, n_rows - r0)))
        return self.results


@dataclass
class CompactResult:
    before: List[DataFileMeta] = field(default_factory=list)
    after: List[DataFileMeta] = field(default_factory=list)
    written: List[WrittenFile] = field(default_factory=list)


class MergeTreeCompactRewriter:
    """rewriteCompaction(outputLevel, dropDelete, sections): every section is merged on the device, the merged
    batch never leaves HBM before it is encoded (MergeTreeCompactRewriter.java:78-116).  With `options` (table
    options), the files written at the output level take the format format_for_level(options, level) and, for
    parquet, the codec compression_for_level(options, level), for orc orc_compression_for_level(options, level),
    and the 'file-index.*' options give every file its bloom filters (refused before any device work when the device
    cannot build them); without, they are uncompressed Parquet (or the writer arguments' file_format).  With
    `page_index` the files of Parquet output levels carry the page index (ColumnIndex and OffsetIndex); ORC output
    levels ignore it.  With `row_index` the files of ORC output levels carry a row index and bloom filters as the
    table options ask for them (orc_index_for_level); Parquet output levels ignore it.  The files of Parquet output
    levels carry the Parquet bloom filters the table options ask for (parquet_bloom_for_level)."""

    def __init__(self, schema: KeyValueSchema, mf_factory: MergeFunctionFactory, directory: str,
                 user_defined_seq_comparator=None, file_io: Optional[LocalFileIO] = None, device: int = 0,
                 target_file_rows: int = 4 << 20, options: Optional[Dict[str, object]] = None,
                 page_index: bool = False, row_index: bool = False, **writer_args):
        self.schema = schema
        self.mf_factory = mf_factory
        self.directory = directory
        self.udsc = user_defined_seq_comparator
        self.reader_factory = KeyValueFileReaderFactory(schema, file_io, device)
        self.file_io = file_io
        self.device = device
        self.target_file_rows = target_file_rows
        self.options = options
        self.page_index = page_index
        self.row_index = row_index
        self.writer_args = writer_args

    def rewrite(self, output_level: int, drop_delete: bool, sections: Sequence[Sequence[SortedRun]]) -> CompactResult:
        return self.rewrite_compaction(output_level, drop_delete, sections)

    def rewrite_compaction(self, output_level: int, drop_delete: bool,
                           sections: Sequence[Sequence[SortedRun]]) -> CompactResult:
        result = CompactResult()
        spec = self.mf_factory.create().with_drop_delete(drop_delete)
        writer_args = dict(self.writer_args)
        if self.options is not None:
            fmt = format_for_level(self.options, output_level)
            if fmt not in FILE_FORMATS:
                raise N.UnsupportedOnDevice(2, f"file format '{fmt}' of level {output_level} is not written on the "
                                               f"device (parquet and orc are)")
            writer_args["file_format"] = fmt
            if fmt == "orc":
                (writer_args["compression"], writer_args["zstd_level"],
                 writer_args["compression_block_size"]) = orc_compression_for_level(self.options, output_level)
            else:
                writer_args["compression"], writer_args["zstd_level"] = compression_for_level(self.options, output_level)
                writer_args["parquet_bloom"] = parquet_bloom_for_level(self.schema, self.options)
            file_index = FileIndexOptions.from_options(self.options)
            if not file_index.is_empty():
                DataFileIndexWriter(self.schema, file_index)          # refuses before any device work
                writer_args["file_index"] = file_index
        parquet = writer_args.get("file_format", "parquet").lower() == "parquet"
        if self.row_index and not parquet:
            writer_args.update(orc_index_for_level(self.options))
            orc_index_options(self.schema, writer_args["row_index_stride"], writer_args["bloom_filter_columns"],
                              writer_args.get("bloom_filter_fpp", 0.01))   # refuses before any device work
        rolling = RollingFileWriter(self.schema, self.directory, output_level, self.target_file_rows, self.file_io,
                                    prefix=f"compact-l{output_level}", page_index=self.page_index and parquet,
                                    **writer_args)
        for section in sections:
            for run in section:
                result.before += run.files
            runs = MergeTreeReaders.open_runs(section, self.reader_factory)
            try:
                merge = SortMergeReader.create_sort_merge_reader(runs, None, self.udsc, spec, device=self.device)
            except Exception:
                for r in runs:
                    r.close()
                raise
            try:
                merge.execute()
                n_out = merge.device_batch().n_rows
                if n_out:
                    rolling.write(merge._merge_h, n_out)
            finally:
                merge.close()
        result.written = rolling.results
        result.after = [w.meta for w in rolling.results]
        return result

    @staticmethod
    def sections_of(files: Sequence[DataFileMeta]) -> List[List[SortedRun]]:
        return IntervalPartition(files).partition()
