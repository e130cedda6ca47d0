"""The data-file index of the compaction output: bloom filters over value columns, built on the device.

Mirrors (same names, same argument meaning):
  FileIndexOptions                 paimon-api/.../fileindex/FileIndexOptions.java:55-140
  MemorySize.parseBytes            paimon-api/.../options/MemorySize.java:280-345
  FileIndexFormat.Writer           paimon-common/.../fileindex/FileIndexFormat.java:127-233
  DataFileIndexWriter              paimon-core/.../io/DataFileIndexWriter.java:70-195
  BloomFilterFileIndex             paimon-common/.../fileindex/bloomfilter/BloomFilterFileIndex.java

The filters themselves (hash of every non-NULL value, bit positions) are built by pg_bloom_filter_build over the rows of
the file, in HBM; the host only lays the per-column bytes into the FileIndexFormat container and decides between the
embedded bytes of DataFileMeta and a side file '<data file>.index' (KeyValueDataFileWriter.java:156-181).
"""
from __future__ import annotations

import ctypes as C
import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import _native as N
from .types import KeyValueSchema, type_root

FILE_INDEX_PREFIX = "file-index."
COLUMNS_SUFFIX = ".columns"
IN_MANIFEST_THRESHOLD = "file-index.in-manifest-threshold"
DEFAULT_IN_MANIFEST_THRESHOLD = "500 B"           # CoreOptions.FILE_INDEX_IN_MANIFEST_THRESHOLD
INDEX_PATH_SUFFIX = ".index"                      # DataFilePathFactory.INDEX_PATH_SUFFIX
BLOOM_FILTER = "bloom-filter"
BLOOM_DEFAULT_ITEMS, BLOOM_DEFAULT_FPP = 1_000_000, 0.1
MAGIC = 1493475289347502
VERSION = 1

_UNITS = {"b": 1, "bytes": 1, "k": 1 << 10, "kb": 1 << 10, "kibibytes": 1 << 10, "m": 1 << 20, "mb": 1 << 20,
          "mebibytes": 1 << 20, "g": 1 << 30, "gb": 1 << 30, "gibibytes": 1 << 30, "t": 1 << 40, "tb": 1 << 40,
          "tebibytes": 1 << 40}


def parse_memory_size(text) -> int:
    """MemorySize.parseBytes: a decimal number of bytes with an optional binary unit (b, k / kb, m / mb, g / gb,
    t / tb, or their long names), case-insensitive, blanks around either part allowed."""
    t = str(text).strip()
    if not t:
        raise ValueError("argument is an empty- or whitespace-only string")
    pos = 0
    while pos < len(t) and "0" <= t[pos] <= "9":
        pos += 1
    number, unit = t[:pos], t[pos:].strip().lower()
    if not number:
        raise ValueError("text does not start with a number")
    value = int(number)
    if value >= 1 << 63:
        raise ValueError(f"The value '{number}' cannot be re represented as 64bit number (numeric overflow).")
    if unit and unit not in _UNITS:
        raise ValueError(f"Memory size unit '{unit}' does not match any of the recognized units")
    result = value * _UNITS.get(unit, 1)
    if result >= 1 << 63:
        raise ValueError(f"The value '{text}' cannot be re represented as 64bit number of bytes (numeric overflow).")
    return result


def _int32(x: int) -> int:
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x & 0x80000000 else x


def java_string_hash(s: str) -> int:
    """String.hashCode over the UTF-16 code units."""
    h = 0
    units = s.encode("utf-16-be")
    for i in range(0, len(units), 2):
        h = (31 * h + (units[i] << 8 | units[i + 1])) & 0xFFFFFFFF
    return _int32(h)


def _column_hash(column: str) -> int:
    """FileIndexOptions.Column.hashCode: Arrays.hashCode({name, null, false}) of a top-level column,
    Arrays.hashCode({name, key, true}) of 'name[key]'."""
    if is_nested(column):
        i = column.index("[")
        return _int32(((31 + java_string_hash(column[:i])) * 31 + java_string_hash(column[i + 1:-1])) * 31 + 1231)
    return _int32(((31 + java_string_hash(column)) * 31 + 0) * 31 + 1237)


class _JavaHashMap:
    """The iteration order of a java.util.HashMap's keys: tables of 16 << n buckets, resized when they hold more than
    3/4 of that, bucket (h ^ h >>> 16) & (size - 1); put() appends to a bucket and resizes after inserting,
    computeIfAbsent() resizes before and puts a new key at the head of its bucket.  (Buckets of 8 or more keys turn
    into trees; the few column names of a file index never get there.)"""

    def __init__(self, hash_fn):
        self._hash = hash_fn
        self._table: Optional[List[list]] = None
        self._size = 0

    def _bucket(self, key) -> list:
        h = self._hash(key) & 0xFFFFFFFF
        return self._table[(h ^ (h >> 16)) & (len(self._table) - 1)]

    def _resize(self) -> None:
        old = self._table or []
        self._table = [[] for _ in range(2 * len(old) if old else 16)]
        for b in old:
            for k in b:
                self._bucket(k).append(k)

    def _threshold(self) -> int:
        return len(self._table) * 3 // 4

    def put(self, key) -> None:
        if self._table is None:
            self._resize()
        b = self._bucket(key)
        if key not in b:
            b.append(key)
            self._size += 1
            if self._size > self._threshold():
                self._resize()

    def compute_if_absent(self, key) -> None:
        if self._table is None or self._size > self._threshold():
            self._resize()
        b = self._bucket(key)
        if key not in b:
            b.insert(0, key)
            self._size += 1

    def keys(self) -> list:
        return [k for b in (self._table or []) for k in b]


def _split(text: str, sep: str) -> List[str]:
    """String.split: trailing empty strings are dropped."""
    parts = text.split(sep)
    while parts and parts[-1] == "":
        parts.pop()
    return parts


def is_nested(column: str) -> bool:
    """FileIndexOptions.topLevelIndexOfNested: 'm[key]' names the values of map column m under key."""
    return column.find("[") != -1 and column.endswith("]")


def top_level(column: str) -> str:
    return column[:column.index("[")] if is_nested(column) else column


@dataclass
class FileIndexOptions:
    """The 'file-index.*' table options: columns[column][index type] = that index's options of the column, the columns in
    the order the reference's option map iterates them; in_manifest_threshold in bytes."""
    columns: Dict[str, Dict[str, Dict[str, str]]] = field(default_factory=dict)
    in_manifest_threshold: int = 500

    @staticmethod
    def from_options(options: Optional[Dict[str, object]]) -> "FileIndexOptions":
        options = {str(k): str(v) for k, v in (options or {}).items()}
        order = _JavaHashMap(_column_hash)
        columns: Dict[str, Dict[str, Dict[str, str]]] = {}
        rest = {}
        for key, value in options.items():
            if not key.startswith(FILE_INDEX_PREFIX):
                continue
            if key.endswith(COLUMNS_SUFFIX):
                index_type = key[len(FILE_INDEX_PREFIX):len(key) - len(COLUMNS_SUFFIX)]
                for name in _split(value, ","):
                    if not name.strip():
                        raise ValueError(f"Wrong option in {key}, should not have empty column")
                    name = name.strip()
                    order.compute_if_absent(name)
                    columns.setdefault(name, {}).setdefault(index_type, {})
            else:
                rest[key] = value
        for key, value in rest.items():
            kv = _split(key[len(FILE_INDEX_PREFIX):], ".")
            if len(kv) != 3:                       # options that are not <type>.<column>.<option> are ignored
                continue
            index_type, cname, opt = kv
            if index_type in columns.get(cname, {}):
                columns[cname][index_type][opt] = value
            elif not any(is_nested(c) and top_level(c) == cname and index_type in t for c, t in columns.items()):
                # (an option of map column m itself applies to its 'm[key]' indexes, which are refused later)
                raise ValueError(f"Can't find top level column options for map type: {cname} {index_type}")
        threshold = parse_memory_size(options.get(IN_MANIFEST_THRESHOLD, DEFAULT_IN_MANIFEST_THRESHOLD))
        return FileIndexOptions({name: columns[name] for name in order.keys()}, threshold)

    def is_empty(self) -> bool:
        return not self.columns


def write_utf(s: str) -> bytes:
    """DataOutputStream.writeUTF: a big-endian u16 byte count, then modified UTF-8 (U+0000 as two bytes, each UTF-16
    unit of a surrogate pair as three)."""
    units = s.encode("utf-16-be")
    out = bytearray()
    for i in range(0, len(units), 2):
        c = units[i] << 8 | units[i + 1]
        if 0 < c < 0x80:
            out.append(c)
        elif c < 0x800:
            out += bytes((0xC0 | c >> 6, 0x80 | c & 0x3F))
        else:
            out += bytes((0xE0 | c >> 12, 0x80 | c >> 6 & 0x3F, 0x80 | c & 0x3F))
    if len(out) > 0xFFFF:
        raise ValueError(f"encoded string too long: {len(out)} bytes")
    return struct.pack(">H", len(out)) + bytes(out)


def serialize_file_index(indexes: Dict[str, Dict[str, bytes]]) -> bytes:
    """FileIndexFormat.Writer.writeColumnIndexes: magic, version, head length, column count; per column its name, index
    count and per index its type, start (from the file's first byte) and length; a redundant length of 0; the bodies.
    Big-endian throughout; columns and index types in the order of `indexes`."""
    names = b"".join(write_utf(c) + b"".join(write_utf(t) for t in types) for c, types in indexes.items())
    n_indexes = sum(len(types) for types in indexes.values())
    head_length = 8 + 4 + 4 + 4 + 8 * n_indexes + 4 * len(indexes) + 4 + len(names)
    head = bytearray(struct.pack(">qii", MAGIC, VERSION, head_length) + struct.pack(">i", len(indexes)))
    body = bytearray()
    for column, types in indexes.items():
        head += write_utf(column) + struct.pack(">i", len(types))
        for index_type, data in types.items():
            head += write_utf(index_type) + struct.pack(">ii", head_length + len(body), len(data))
            body += data
    head += struct.pack(">i", 0)
    assert len(head) == head_length
    return bytes(head + body)


@dataclass
class FileIndexResult:
    embedded_index: Optional[bytes] = None        # DataFileMeta.embeddedIndex
    extra_files: List[str] = field(default_factory=list)


class DataFileIndexWriter:
    """The index of one data file of `schema` (its value fields, as KeyValueDataFileWriter indexes kv.value()).  The
    constructor resolves the options against the value type and refuses what the device does not build or the
    reference does not allow, so that a writer fails before any device work:
      - index types other than bloom-filter, and map-value columns 'm[key]': UnsupportedOnDevice;
      - a column the value type lacks: '<col> does not exist in column fields' (DataFileIndexWriter.java:98-101);
      - BOOLEAN and DECIMAL columns: 'Does not support type boolean' / 'Does not support decimal' (FastHash.java)."""

    def __init__(self, schema: KeyValueSchema, options: FileIndexOptions):
        self.threshold = options.in_manifest_threshold
        fields = {f.name: (i, f) for i, f in enumerate(schema.value_type.fields)}
        maintainers = _JavaHashMap(java_string_hash)      # DataFileIndexWriter's column -> maintainer of the type
        specs: Dict[str, Tuple[int, int, float]] = {}
        for column, types in options.columns.items():
            name = top_level(column)
            if name not in fields:
                raise ValueError(f"{name} does not exist in column fields")
            for index_type, opts in types.items():
                if index_type != BLOOM_FILTER:
                    raise N.UnsupportedOnDevice(2, f"file index type '{index_type}' of column {column} is not built on "
                                                   f"the device (bloom-filter is)")
                if is_nested(column):
                    raise N.UnsupportedOnDevice(2, f"file index on the map values {column} is not built on the device")
                idx, f = fields[name]
                root = type_root(f.type)
                if root == "BOOLEAN":
                    raise ValueError("Does not support type boolean")
                if root == "DECIMAL":
                    raise ValueError("Does not support decimal")
                items = int(opts.get("items", BLOOM_DEFAULT_ITEMS))
                fpp = float(opts.get("fpp", BLOOM_DEFAULT_FPP))
                if not 0 < items < 1 << 31 or not 0 < fpp < 1:
                    raise ValueError(f"bloom filter of {column}: items must be in [1, 2^31) and fpp in (0, 1), got "
                                     f"items {items}, fpp {fpp}")
                maintainers.put(column)
                specs[column] = (schema.n_key + 2 + idx, items, fpp)
        order = _JavaHashMap(java_string_hash)            # serializeMaintainers' column -> bytes
        for column in maintainers.keys():
            order.compute_if_absent(column)
        self.columns = order.keys()
        self.specs = [specs[c] for c in self.columns]
        self.lib = N.load()
        self.sizes = []
        for column, (_, items, fpp) in zip(self.columns, self.specs):
            size = C.c_int64(0)
            N.check(self.lib.pg_bloom_filter_size(items, fpp, C.byref(size), None))
            self.sizes.append(size.value)

    def build(self, source_handle: int, row0: int = 0, n_rows: int = -1) -> Dict[str, bytes]:
        """The serialized bloom filter of every indexed column over rows [row0, row0 + n_rows) of a merge or run
        handle, in the container's column order."""
        n = len(self.specs)
        specs = (N.PgBloomFilterSpec * n)(*[N.PgBloomFilterSpec(*s) for s in self.specs])
        bufs = [np.empty(size, np.uint8) for size in self.sizes]
        outs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
        caps = (C.c_int64 * n)(*self.sizes)
        N.check(self.lib.pg_bloom_filter_build(source_handle, row0, n_rows, n, specs, outs, caps))
        return {c: b.tobytes() for c, b in zip(self.columns, bufs)}

    def write(self, file_io, data_path: str, source_handle: int, row0: int = 0, n_rows: int = -1) -> FileIndexResult:
        """DataFileIndexWriter.close / result for the file at `data_path`: the container as embedded bytes when it is at
        most the in-manifest threshold, else written to '<data_path>.index' through `file_io`."""
        data = serialize_file_index({c: {BLOOM_FILTER: b} for c, b in self.build(source_handle, row0, n_rows).items()})
        if len(data) <= self.threshold:
            return FileIndexResult(embedded_index=data)
        file_io.write_bytes(data_path + INDEX_PATH_SUFFIX, data)
        return FileIndexResult(extra_files=[data_path + INDEX_PATH_SUFFIX])
