"""Plain numpy restatement of the statistics a compaction output file carries.  TEST INFRASTRUCTURE ONLY.

The device encoder (paimon_b200/csrc/parquet_encode.cu) writes statistics at two levels, and every later reader
prunes row groups and files with them:
  * per row group and column, the Parquet footer `Statistics`: null_count, min_value, max_value;
  * per file and column, SimpleColStats(min, max, null_count), plus the DataFileMeta fields row count, min / max
    sequence number, delete row count and min / max key.
Nothing here calls the library; the rules below are written from the sources they cite.

Row groups follow the encoder's cut: page_rows (default 32768) is rounded up to a multiple of 8, row_group_rows
(default 2^20) up to a multiple of page_rows, and the groups of a slice [row0, row0 + n) start at row0.

Rules:
  * Integers, DATE, TIME, TIMESTAMP, DECIMAL (the unscaled value) and BOOLEAN: numeric min and max of the non-null
    values.  The footer holds the physical value: TINYINT and SMALLINT sign-extended to a 4-byte INT32, INT32 as 4
    bytes, INT64 (BIGINT, TIMESTAMP, DECIMAL) as 8 bytes, BOOLEAN as 1 byte.
  * FLOAT and DOUBLE per row group (parquet.thrift, `Statistics`, on min_value / max_value of floating point
    columns): a chunk with a NaN among its non-null values has no min / max; otherwise numeric min and max, where a
    zero min is written as -0.0 and a zero max as +0.0.  pyarrow's writer applies the same zero rule.
  * FLOAT and DOUBLE per file: no min / max if any non-null value of the file is NaN; otherwise the merge of the row
    groups, the zero rule again.  This is a choice made for soundness: Paimon merges the footer statistics of a file
    with parquet-mr's Statistics.mergeStatistics (paimon-format/.../parquet/ParquetUtil.java:70-89), and what
    parquet-mr does with NaN is not in the Paimon sources.  Paimon's predicates compare with Comparable.compareTo
    (paimon-common/.../predicate/CompareUtils.java:29-31), i.e. Double.compare: -0.0 < +0.0, NaN above +inf.  A
    file that held a NaN but reported a finite max would be skipped by `x > max`, although the NaN row matches.
  * STRING and BINARY: no min / max in the footer and (None, None, null_count) at the file level.  This pins what
    the encoder writes today; Paimon's truncated string statistics are not written.
  * A column without non-null values has no min / max; its null count is its row count.
  * DataFileMeta (paimon-core/.../io/KeyValueDataFileWriter.java:108-184): row_count; min / max of
    _SEQUENCE_NUMBER; delete_row_count = rows whose _VALUE_KIND is a retract, UPDATE_BEFORE (1) or DELETE (3)
    (:124-126); min_key / max_key = the key of the first and of the last row (:116-119, :166-167), a scalar for a
    one-field key, else a tuple.
"""
from __future__ import annotations

import struct
from typing import List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from paimon_b200.columnar import KeyValueBatch
from paimon_b200.types import PhysicalType

_FLOATS = (PhysicalType.FLOAT, PhysicalType.DOUBLE)
_VARLEN = (PhysicalType.STRING, PhysicalType.BINARY)
_RETRACT_KINDS = (1, 3)                                       # RowKind.UPDATE_BEFORE, RowKind.DELETE


class ChunkStats(NamedTuple):
    """The footer Statistics of one column chunk; min / max are the footer bytes, None when not written."""
    null_count: int
    min: Optional[bytes]
    max: Optional[bytes]

    @property
    def has_min_max(self) -> bool:
        return self.min is not None


class FileColStats(NamedTuple):
    """SimpleColStats of one column of a file: Python int / float / bool, or None."""
    min: object
    max: object
    null_count: int


class FileMeta(NamedTuple):
    row_count: int
    min_sequence_number: Optional[int]
    max_sequence_number: Optional[int]
    delete_row_count: int
    min_key: object
    max_key: object


# ---------------------------------------------------------------------------------------------- comparisons

def _double_to_long_bits(x: float) -> int:
    """Double.doubleToLongBits: every NaN collapses to 0x7ff8000000000000."""
    if x != x:
        return 0x7FF8000000000000
    return struct.unpack("<q", struct.pack("<d", x))[0]


def java_compare(a, b) -> int:
    """Double.compare(a, b) for floats (-0.0 < +0.0; NaN equals NaN and is above +inf), Long.compare for ints."""
    if isinstance(a, (float, np.floating)) or isinstance(b, (float, np.floating)):
        a, b = float(a), float(b)
        if a < b:
            return -1
        if a > b:
            return 1
        x, y = _double_to_long_bits(a), _double_to_long_bits(b)
        return (x > y) - (x < y)
    a, b = int(a), int(b)
    return (a > b) - (a < b)


# ---------------------------------------------------------------------------------------------- layout

def writer_rows(page_rows: int = 0, row_group_rows: int = 0) -> Tuple[int, int]:
    """(page rows, row-group rows) as the encoder rounds them (parquet_encode.cu, make_plan())."""
    page = page_rows if page_rows > 0 else 32768
    page = (page + 7) & ~7
    group = row_group_rows if row_group_rows > 0 else 1 << 20
    group = -(-group // page) * page
    return page, group


def row_groups(n_rows: int, page_rows: int = 0, row_group_rows: int = 0) -> List[Tuple[int, int]]:
    """[start, stop) of every row group, relative to the first row of the slice."""
    _, group = writer_rows(page_rows, row_group_rows)
    return [(g, min(n_rows, g + group)) for g in range(0, n_rows, group)]


def _slice(batch: KeyValueBatch, row0: int, n_rows: int) -> Tuple[int, int]:
    if n_rows < 0:
        n_rows = batch.n_rows - row0
    assert 0 <= row0 and row0 + n_rows <= batch.n_rows
    return row0, n_rows


def _valid(col, start: int, stop: int) -> np.ndarray:
    if col.valid is None:
        return np.ones(stop - start, bool)
    bits = np.unpackbits(np.asarray(col.valid, np.uint8), bitorder="little")
    return bits[start:stop].astype(bool)


def non_null_values(col, start: int, stop: int) -> np.ndarray:
    """The non-null values of rows [start, stop) (fixed-width columns)."""
    return np.asarray(col.data[start:stop])[_valid(col, start, stop)]


# ---------------------------------------------------------------------------------------------- the rules

def footer_bytes(t: PhysicalType, v) -> bytes:
    """A min / max value as the footer stores it for a column of physical type t."""
    t = PhysicalType(t)
    if t in (PhysicalType.INT8, PhysicalType.INT16, PhysicalType.INT32):
        return struct.pack("<i", int(v))
    if t == PhysicalType.INT64:
        return struct.pack("<q", int(v))
    if t == PhysicalType.FLOAT:
        return np.float32(v).tobytes()
    if t == PhysicalType.DOUBLE:
        return np.float64(v).tobytes()
    if t == PhysicalType.BOOL:
        return bytes([int(bool(v))])
    raise ValueError(f"no footer min / max for {t!r}")


def _min_max(t: PhysicalType, vals: np.ndarray):
    """(min, max) of the non-null values of a chunk or file, numpy scalars, or None when none may be written."""
    if t in _VARLEN or len(vals) == 0:
        return None
    if t in _FLOATS:
        if np.isnan(vals).any():
            return None
        lo, hi = vals.min(), vals.max()
        dt = vals.dtype.type
        return (dt(-0.0) if lo == 0 else lo), (dt(0.0) if hi == 0 else hi)
    if t == PhysicalType.BOOL:
        vals = vals != 0
    return vals.min(), vals.max()


def chunk_stats(batch: KeyValueBatch, c: int, start: int, stop: int) -> ChunkStats:
    """The footer Statistics of column c over rows [start, stop) of the batch."""
    t = batch.schema.physical_types()[c]
    col = batch.columns[c]
    valid = _valid(col, start, stop)
    nulls = int((~valid).sum())
    mm = None if t in _VARLEN else _min_max(t, non_null_values(col, start, stop))
    if mm is None:
        return ChunkStats(nulls, None, None)
    return ChunkStats(nulls, footer_bytes(t, mm[0]), footer_bytes(t, mm[1]))


def footer_stats(batch: KeyValueBatch, row0: int = 0, n_rows: int = -1, page_rows: int = 0,
                 row_group_rows: int = 0) -> List[List[ChunkStats]]:
    """[row group][column] footer statistics of the file the encoder writes for rows [row0, row0 + n_rows)."""
    row0, n_rows = _slice(batch, row0, n_rows)
    return [[chunk_stats(batch, c, row0 + a, row0 + b) for c in range(batch.schema.n_cols)]
            for a, b in row_groups(n_rows, page_rows, row_group_rows)]


def _py(t: PhysicalType, v):
    if t in _FLOATS:
        return float(v)
    if t == PhysicalType.BOOL:
        return bool(v)
    return int(v)


def file_stats(batch: KeyValueBatch, row0: int = 0, n_rows: int = -1) -> List[FileColStats]:
    """SimpleColStats of every file column (keys, _SEQUENCE_NUMBER and _VALUE_KIND included).  The row groups
    do not show: for every type the merge of the row groups' statistics is the rule applied to the whole file."""
    row0, n_rows = _slice(batch, row0, n_rows)
    out = []
    for c, t in enumerate(batch.schema.physical_types()):
        col = batch.columns[c]
        nulls = int((~_valid(col, row0, row0 + n_rows)).sum())
        mm = None if t in _VARLEN else _min_max(t, non_null_values(col, row0, row0 + n_rows))
        out.append(FileColStats(None, None, nulls) if mm is None else FileColStats(_py(t, mm[0]), _py(t, mm[1]), nulls))
    return out


def _key_row(batch: KeyValueBatch, row: int):
    vals = []
    for i in range(batch.schema.n_key):
        col = batch.columns[i]
        if col.offsets is not None:
            b = np.asarray(col.data[col.offsets[row]:col.offsets[row + 1]]).tobytes()
            vals.append(b.decode() if PhysicalType(col.type) == PhysicalType.STRING else b)
        else:
            vals.append(col.data[row].item())
    return vals[0] if len(vals) == 1 else tuple(vals)


def data_file_meta(batch: KeyValueBatch, row0: int = 0, n_rows: int = -1) -> FileMeta:
    """The DataFileMeta fields of the file holding rows [row0, row0 + n_rows); None where an empty file has none."""
    row0, n_rows = _slice(batch, row0, n_rows)
    nk = batch.schema.n_key
    seq = np.asarray(batch.columns[nk].data[row0:row0 + n_rows], np.int64)
    kinds = np.asarray(batch.columns[nk + 1].data[row0:row0 + n_rows])
    if n_rows == 0:
        return FileMeta(0, None, None, 0, None, None)
    return FileMeta(n_rows, int(seq.min()), int(seq.max()), int(np.isin(kinds, _RETRACT_KINDS).sum()),
                    _key_row(batch, row0), _key_row(batch, row0 + n_rows - 1))


# ---------------------------------------------------------------------------------------------- soundness

def value_of(t: PhysicalType, b: bytes):
    """Footer bytes back to a Python value (the inverse of footer_bytes)."""
    t = PhysicalType(t)
    if t in (PhysicalType.INT8, PhysicalType.INT16, PhysicalType.INT32):
        return struct.unpack("<i", b)[0]
    if t == PhysicalType.INT64:
        return struct.unpack("<q", b)[0]
    if t == PhysicalType.FLOAT:
        return float(np.frombuffer(b, np.float32)[0])
    if t == PhysicalType.DOUBLE:
        return float(np.frombuffer(b, np.float64)[0])
    return bool(b[0])


def unsound(t: PhysicalType, lo, hi, vals: Sequence) -> list:
    """The non-null values v of a chunk or file for which min <= v <= max does not hold under Double.compare /
    Long.compare (empty when the statistics are sound).  lo / hi are Python values, None = not written."""
    if lo is None and hi is None:
        return []
    if lo is None or hi is None:
        return ["min / max half written"]
    t = PhysicalType(t)
    bad = []
    distinct = {np.asarray(v).tobytes(): v for v in np.asarray(vals)}.values()   # NaN payloads and zeros kept apart
    for v in distinct:
        pv = float(v) if t in _FLOATS else int(v)
        if java_compare(lo, pv) > 0 or java_compare(pv, hi) > 0:
            bad.append(pv)
    return bad
