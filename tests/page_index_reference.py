"""Plain-Python restatement of the Parquet page index a compaction output file carries.  TEST INFRASTRUCTURE ONLY.

With pg_parquet_write_options.page_index = 1 the device encoder (paimon_b200/csrc/parquet_encode.cu) writes, for
every column chunk, the two structures of parquet.thrift that parquet-mr writes and that the Parquet reader Paimon
vendors uses to skip pages inside a row group (paimon-format/.../parquet/hadoop/ParquetFileReader.java:368-375,
558-617):
  * ColumnIndex {1: null_pages list<bool>, 2: min_values list<binary>, 3: max_values list<binary>,
    4: boundary_order BoundaryOrder, 5: null_counts list<i64>}
  * OffsetIndex {1: page_locations list<PageLocation {1: offset i64, 2: compressed_page_size i32,
    3: first_row_index i64}>}
Nothing here calls the library; the rules below are written from the format and from parquet-mr's behaviour.

Rules:
  * Pages are the encoder's (stats_reference.writer_rows): each row group is cut into pages of page_rows rows.
  * A page whose rows are all NULL is a null page: null_pages = true, empty min and max.
  * Fixed-width bounds are PLAIN-encoded in the physical type, as the footer's chunk Statistics are
    (stats_reference.footer_bytes): INT8 / INT16 / INT32 as 4 bytes, INT64 8, BOOLEAN 1, FLOAT 4, DOUBLE 8.
    FLOAT / DOUBLE: a zero min is written as -0.0, a zero max as +0.0, per page.  A chunk with a NaN among the
    non-null values of any page has no ColumnIndex (parquet-mr invalidates such a column index); its OffsetIndex
    is still written.
  * STRING / BINARY bounds are the least and greatest non-null value in unsigned-byte order (a proper prefix
    first), truncated to 64 bytes (parquet-mr's default truncation length): a value of at most 64 bytes whole; a
    longer min its 64-byte prefix (STRING: cut back to a code-point boundary); a longer max that prefix up to its last
    position that can be incremented, incremented (BINARY: the last byte below 0xFF; STRING: the last code point
    below U+10FFFF, the surrogate range skipped); when there is none, the whole value.
  * boundary_order over the non-null pages, on the bounds as written, in the column's order (signed integers,
    numeric floats, unsigned bytes): ASCENDING (1) if the mins and the maxes are both non-decreasing, else
    DESCENDING (2) if both are non-increasing, else UNORDERED (0).  At most one non-null page: ASCENDING.
  * OffsetIndex: offset = file offset of the page header, compressed_page_size = header bytes + stored bytes,
    first_row_index relative to the row group's first row.
  * Layout: after the last row group every ColumnIndex (row group major, then column), then every OffsetIndex, then
    the footer; ColumnChunk fields 4 / 5 (offset_index_offset / _length) and 6 / 7 (column_index_offset / _length)
    point at them, 6 / 7 absent where there is no ColumnIndex.
"""
from __future__ import annotations

import struct
from typing import Dict, List, NamedTuple, Optional, Tuple

import numpy as np

import stats_reference as S
from paimon_b200.columnar import KeyValueBatch
from paimon_b200.types import PhysicalType

TRUNCATE = 64
UNORDERED, ASCENDING, DESCENDING = 0, 1, 2
_FLOATS = (PhysicalType.FLOAT, PhysicalType.DOUBLE)
_VARLEN = (PhysicalType.STRING, PhysicalType.BINARY)


class ColumnIndex(NamedTuple):
    null_pages: List[bool]
    min_values: List[bytes]
    max_values: List[bytes]
    boundary_order: int
    null_counts: List[int]


class ChunkIndex(NamedTuple):
    """The page index of one column chunk: its ColumnIndex (None: not written) and each page's (first row in the
    row group, rows)."""
    column_index: Optional[ColumnIndex]
    pages: List[Tuple[int, int]]


# ---------------------------------------------------------------------------------------------- truncation

def truncate_min(v: bytes, utf8: bool) -> bytes:
    if len(v) <= TRUNCATE:
        return v
    n = TRUNCATE
    if utf8:
        while n > 0 and (v[n] & 0xC0) == 0x80:
            n -= 1
    return v[:n]


def truncate_max(v: bytes, utf8: bool) -> bytes:
    if len(v) <= TRUNCATE:
        return v
    if not utf8:
        p = v[:TRUNCATE]
        for i in range(len(p) - 1, -1, -1):
            if p[i] != 0xFF:
                return p[:i] + bytes([p[i] + 1])
        return v
    chars = truncate_min(v, True).decode("utf-8")
    for i in range(len(chars) - 1, -1, -1):
        cp = ord(chars[i])
        if cp < 0x10FFFF:
            cp += 1
            if 0xD800 <= cp <= 0xDFFF:
                cp = 0xE000
            return (chars[:i] + chr(cp)).encode("utf-8")
    return v


# ---------------------------------------------------------------------------------------------- order

def bound_value(t: PhysicalType, b: bytes):
    """A written bound as a value of the column's order."""
    t = PhysicalType(t)
    if t in _VARLEN:
        return bytes(b)
    return S.value_of(t, b)


def boundary_order(t: PhysicalType, null_pages: List[bool], mins: List[bytes], maxs: List[bytes]) -> int:
    lo = [bound_value(t, m) for m, n in zip(mins, null_pages) if not n]
    hi = [bound_value(t, m) for m, n in zip(maxs, null_pages) if not n]
    pairs = list(zip(zip(lo, lo[1:]), zip(hi, hi[1:])))
    if all(a <= b and c <= d for (a, b), (c, d) in pairs):
        return ASCENDING
    if all(a >= b and c >= d for (a, b), (c, d) in pairs):
        return DESCENDING
    return UNORDERED


# ---------------------------------------------------------------------------------------------- the rules

def _valid(col, start: int, stop: int) -> np.ndarray:
    if col.valid is None:
        return np.ones(stop - start, bool)
    return np.unpackbits(np.asarray(col.valid, np.uint8), bitorder="little")[start:stop].astype(bool)


def varlen_values(col, start: int, stop: int) -> List[bytes]:
    """The non-null values of rows [start, stop) of a STRING / BINARY column, as bytes."""
    data = np.asarray(col.data, np.uint8)
    off = np.asarray(col.offsets)
    valid = _valid(col, start, stop)
    return [data[off[r]:off[r + 1]].tobytes() for r in range(start, stop) if valid[r - start]]


def page_entry(batch: KeyValueBatch, c: int, start: int, stop: int) -> Tuple[bool, bytes, bytes, int, bool]:
    """(null page, min, max, null count, NaN seen) of column c over rows [start, stop)."""
    t = PhysicalType(batch.schema.physical_types()[c])
    col = batch.columns[c]
    nulls = int((~_valid(col, start, stop)).sum())
    if nulls == stop - start:
        return True, b"", b"", nulls, False
    if t in _VARLEN:
        vals = varlen_values(col, start, stop)
        utf8 = t == PhysicalType.STRING
        return False, truncate_min(min(vals), utf8), truncate_max(max(vals), utf8), nulls, False
    vals = S.non_null_values(col, start, stop)
    if t in _FLOATS and np.isnan(vals).any():
        return False, b"", b"", nulls, True
    lo, hi = S._min_max(t, vals)
    return False, S.footer_bytes(t, lo), S.footer_bytes(t, hi), nulls, False


def pages_of(row0: int, n_rows: int, page_rows: int = 0, row_group_rows: int = 0) -> List[List[Tuple[int, int]]]:
    """[row group] -> [(first row in the batch, rows)] of every page of a chunk of that group."""
    page, _ = S.writer_rows(page_rows, row_group_rows)
    return [[(row0 + p, min(b, p + page) - p) for p in range(a, b, page)]
            for a, b in S.row_groups(n_rows, page_rows, row_group_rows)]


def chunk_index(batch: KeyValueBatch, c: int, pages: List[Tuple[int, int]]) -> ChunkIndex:
    entries = [page_entry(batch, c, r, r + n) for r, n in pages]
    g0 = pages[0][0]
    locs = [(r - g0, n) for r, n in pages]
    if any(e[4] for e in entries):
        return ChunkIndex(None, locs)
    null_pages = [e[0] for e in entries]
    mins, maxs = [e[1] for e in entries], [e[2] for e in entries]
    t = batch.schema.physical_types()[c]
    return ChunkIndex(ColumnIndex(null_pages, mins, maxs, boundary_order(t, null_pages, mins, maxs),
                                  [e[3] for e in entries]), locs)


def page_index(batch: KeyValueBatch, row0: int = 0, n_rows: int = -1, page_rows: int = 0,
               row_group_rows: int = 0) -> List[List[ChunkIndex]]:
    """[row group][column] page index of the file the encoder writes for rows [row0, row0 + n_rows)."""
    if n_rows < 0:
        n_rows = batch.n_rows - row0
    return [[chunk_index(batch, c, pages) for c in range(batch.schema.n_cols)]
            for pages in pages_of(row0, n_rows, page_rows, row_group_rows)]


# ---------------------------------------------------------------------------------------------- Thrift compact reader

def _varint(b: bytes, i: int) -> Tuple[int, int]:
    v = s = 0
    while True:
        x = b[i]
        i += 1
        v |= (x & 0x7F) << s
        s += 7
        if x < 0x80:
            return v, i


def _zigzag(v: int) -> int:
    return (v >> 1) ^ -(v & 1)


def _value(b: bytes, i: int, t: int):
    if t in (1, 2):                                   # a bool list element: one byte, 1 = true
        return b[i] == 1, i + 1
    if t == 3:
        return struct.unpack_from("<b", b, i)[0], i + 1
    if t in (4, 5, 6):
        v, i = _varint(b, i)
        return _zigzag(v), i
    if t == 7:
        return struct.unpack_from("<d", b, i)[0], i + 8
    if t == 8:
        n, i = _varint(b, i)
        return bytes(b[i:i + n]), i + n
    if t in (9, 10):
        h = b[i]
        i += 1
        n, et = h >> 4, h & 0x0F
        if n == 15:
            n, i = _varint(b, i)
        out = []
        for _ in range(n):
            v, i = _value(b, i, et)
            out.append(v)
        return out, i
    if t == 12:
        return read_struct(b, i)
    raise ValueError(f"thrift compact type {t} at {i} not read here")


def read_struct(b: bytes, i: int = 0) -> Tuple[Dict[int, object], int]:
    """A compact-protocol struct at b[i:] -> ({field id: value}, end); structs nest as dicts, lists as lists."""
    fields, last = {}, 0
    while True:
        h = b[i]
        i += 1
        if h == 0:
            return fields, i
        d, t = h >> 4, h & 0x0F
        if d:
            fid = last + d
        else:
            v, i = _varint(b, i)
            fid = _zigzag(v)
        last = fid
        if t in (1, 2):                               # a bool field: the value is the type
            fields[fid] = t == 1
        else:
            fields[fid], i = _value(b, i, t)


def parse_column_index(b: bytes) -> ColumnIndex:
    f, end = read_struct(b)
    assert end == len(b), "trailing bytes after the ColumnIndex"
    return ColumnIndex(f[1], f[2], f[3], f[4], f.get(5))


def parse_offset_index(b: bytes) -> List[Tuple[int, int, int]]:
    """[(offset, compressed_page_size, first_row_index)] of every page."""
    f, end = read_struct(b)
    assert end == len(b), "trailing bytes after the OffsetIndex"
    return [(p[1], p[2], p[3]) for p in f[1]]


class ChunkRefs(NamedTuple):
    """What a footer's ColumnChunk says about its pages and its page index (None: field absent)."""
    data_page_offset: int
    total_compressed_size: int
    num_values: int
    offset_index: Optional[Tuple[int, int]]
    column_index: Optional[Tuple[int, int]]


def footer_chunks(file_bytes: bytes) -> List[List[ChunkRefs]]:
    """[row group][column] ChunkRefs of a whole Parquet file."""
    n = struct.unpack_from("<I", file_bytes, len(file_bytes) - 8)[0]
    start = len(file_bytes) - 8 - n
    fmd, end = read_struct(file_bytes, start)
    assert end == len(file_bytes) - 8
    out = []
    for rg in fmd.get(4, []):
        row = []
        for cc in rg[1]:
            md = cc[3]
            oi = (cc[4], cc[5]) if 4 in cc else None
            ci = (cc[6], cc[7]) if 6 in cc else None
            row.append(ChunkRefs(md[9], md[7], md[5], oi, ci))
        out.append(row)
    return out


def page_header(file_bytes: bytes, off: int) -> Tuple[int, int, int]:
    """(header bytes, compressed_page_size, DataPageHeader.num_values) of the page header at `off`."""
    f, end = read_struct(file_bytes, off)
    return end - off, f[3], f[5][1]
