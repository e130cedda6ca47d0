"""Plain-Python restatement of the Parquet split-block bloom filter (SBBF) a compaction output file carries.  TEST
INFRASTRUCTURE ONLY.

With bloom columns (pg_parquet_encode_bloom) the device encoder (paimon_b200/csrc/parquet_encode.cu) writes one filter
per (row group, bloom column), as parquet-mr writes them for 'parquet.bloom.filter.enabled' (RowDataParquetBuilder.java
:96-116) and as the reader Paimon vendors reads them to drop row groups (ParquetFileReader.java:418-419, 1051-1120).
Nothing here calls the library; the rules are written from the Parquet format specification (BloomFilter.md) and from
parquet-mr 1.16's BlockSplitBloomFilter sizing:
  * Hash: XXH64 (seed 0) of the value's PLAIN bytes: INT8 / INT16 / INT32 / DATE as 4 little-endian bytes
    (sign-extended), INT64 as 8, FLOAT / DOUBLE as their raw IEEE bits (no NaN folding, -0.0 is not +0.0), STRING /
    BINARY as the value bytes without the length word.  NULLs are not inserted.
  * Block: ((h >> 32) * num_blocks) >> 32, blocks of 32 bytes (eight little-endian 32-bit words).
  * Mask: key = h & 0xFFFFFFFF; word i of the block gets bit (key * SALT[i] mod 2^32) >> 27.
  * Sizing: without an ndv the filter has MAX_BYTES (1 MiB, parquet-mr's default, which Paimon does not change).  With
    an ndv: bits = (int)(-8 ndv / ln(1 - fpp^(1/8))), capped at 2^30 bits (the spec's 128 MiB), rounded by
    (bits + 255) & ~256 and floored at 256 bits (optimalNumOfBits); bytes = bits / 8 clamped to [32, MAX_BYTES] and
    rounded up to a power of two.
  * File: ColumnMetaData field 14 (bloom_filter_offset) points at a BloomFilterHeader {1: numBytes, 2: algorithm
    BLOCK{}, 3: hash XXHASH{}, 4: compression UNCOMPRESSED{}}, the bitset follows it; field 15 (bloom_filter_length)
    is header + bitset.
"""
from __future__ import annotations

import math
import struct
from typing import Iterable, List, Optional

import numpy as np
import xxhash

import stats_reference as S
from page_index_reference import _valid, read_struct
from paimon_b200.types import PhysicalType

SALT = (0x47b6137b, 0x44974d91, 0x8824ad5b, 0xa2b7289d, 0x705495c7, 0x2df1424b, 0x9efc4947, 0x5c6bfb31)
MIN_BYTES = 32
MAX_BYTES = 1 << 20
UPPER_BOUND_BYTES = 128 << 20


def num_bytes(ndv: int = 0, fpp: float = 0.01) -> int:
    """The bitset bytes of a filter for `ndv` distinct values at `fpp` (ndv 0: unset, the 1 MiB maximum)."""
    if ndv <= 0:
        return MAX_BYTES
    m = -8 * ndv / math.log(1 - fpp ** (1.0 / 8))
    bits = 2 ** 31 - 1 if m >= 2 ** 31 - 1 else int(m)            # Java's saturating (int) cast
    if bits > UPPER_BOUND_BYTES << 3 or m < 0:
        bits = UPPER_BOUND_BYTES << 3
    bits = max((bits + 255) & ~256, MIN_BYTES << 3)
    n = max(bits // 8, MIN_BYTES)
    if n & (n - 1):
        n = 1 << n.bit_length()
    return min(n, MAX_BYTES)


def plain_bytes(kind: str, v) -> bytes:
    """The PLAIN bytes a value is hashed by.  kind: 'int32' (INT8 / INT16 / INT32 / DATE), 'int64', 'float' and
    'double' (v: the IEEE bits as an int, or a Python float), 'bytes' (str is UTF-8 encoded)."""
    if kind == "int32":
        return struct.pack("<i", int(v))
    if kind == "int64":
        return struct.pack("<q", int(v))
    if kind == "float":
        return struct.pack("<I", v) if isinstance(v, (int, np.integer)) else struct.pack("<f", v)
    if kind == "double":
        return struct.pack("<Q", v) if isinstance(v, (int, np.integer)) else struct.pack("<d", v)
    return v.encode() if isinstance(v, str) else bytes(v)


def hash_value(kind: str, v) -> int:
    return xxhash.xxh64_intdigest(plain_bytes(kind, v), seed=0)


def bitset_of_hashes(hashes: np.ndarray, n_bytes: int) -> bytes:
    """The bitset of a filter of n_bytes holding the uint64 `hashes` (vectorised insert())."""
    words = np.zeros(n_bytes // 4, np.uint32)
    h = np.asarray(hashes, np.uint64)
    blk = ((h >> np.uint64(32)) * np.uint64(n_bytes // 32)) >> np.uint64(32)
    key = h & np.uint64(0xFFFFFFFF)
    for i, salt in enumerate(SALT):
        bit = ((key * np.uint64(salt)) & np.uint64(0xFFFFFFFF)) >> np.uint64(27)
        np.bitwise_or.at(words, (blk * np.uint64(8) + np.uint64(i)).astype(np.int64),
                         (np.uint64(1) << bit).astype(np.uint32))
    return words.astype("<u4").tobytes()


def column_hashes(col, start: int, stop: int) -> np.ndarray:
    """The hashes of the non-NULL values of rows [start, stop) of a batch column (columnar.Column), by its PLAIN
    bytes: INT8 / INT16 widened to INT32."""
    valid = _valid(col, start, stop)
    t = PhysicalType(col.type)
    if t in (PhysicalType.STRING, PhysicalType.BINARY):
        data, off = np.asarray(col.data, np.uint8), np.asarray(col.offsets)
        vals = [data[off[r]:off[r + 1]].tobytes() for r in range(start, stop) if valid[r - start]]
    else:
        v = np.asarray(col.data)[start:stop][valid]
        if t in (PhysicalType.INT8, PhysicalType.INT16):
            v = v.astype(np.int32)
        raw = np.ascontiguousarray(v).tobytes()
        w = v.dtype.itemsize
        vals = [raw[i:i + w] for i in range(0, len(raw), w)]
    return np.array([xxhash.xxh64_intdigest(x) for x in vals], np.uint64)


def file_bitsets(batch, bloom, row0: int = 0, n_rows: int = -1, page_rows: int = 0,
                 row_group_rows: int = 0) -> List[List[Optional[bytes]]]:
    """[row group][column] the bitset the encoder writes for rows [row0, row0 + n_rows) of `batch`, None for a
    column without a filter.  bloom: [(file column, ndv, fpp)]."""
    if n_rows < 0:
        n_rows = batch.n_rows - row0
    size = {c: num_bytes(ndv, fpp) for c, ndv, fpp in bloom}
    return [[bitset_of_hashes(column_hashes(batch.columns[c], row0 + a, row0 + b), size[c]) if c in size else None
             for c in range(batch.schema.n_cols)]
            for a, b in S.row_groups(n_rows, page_rows, row_group_rows)]


def _mask(h: int) -> List[int]:
    key = h & 0xFFFFFFFF
    return [1 << (((key * s) & 0xFFFFFFFF) >> 27) for s in SALT]


def insert(bits: np.ndarray, h: int) -> None:
    """Sets the eight bits of hash h in `bits` (a uint32 array of num_bytes / 4 words)."""
    nb = len(bits) // 8
    blk = ((h >> 32) * nb) >> 32
    for i, m in enumerate(_mask(h)):
        bits[8 * blk + i] |= np.uint32(m)


def find(bits: np.ndarray, h: int) -> bool:
    nb = len(bits) // 8
    blk = ((h >> 32) * nb) >> 32
    return all(int(bits[8 * blk + i]) & m for i, m in enumerate(_mask(h)))


def build(kind: str, values: Iterable, n_bytes: int) -> bytes:
    """The bitset of a filter of n_bytes over the non-None `values`."""
    bits = np.zeros(n_bytes // 4, np.uint32)
    for v in values:
        if v is not None:
            insert(bits, hash_value(kind, v))
    return bits.astype("<u4").tobytes()


def contains(bitset: bytes, kind: str, v) -> bool:
    return find(np.frombuffer(bitset, "<u4"), hash_value(kind, v))


def file_filters(file_bytes: bytes) -> List[List[Optional[dict]]]:
    """[row group][column] of a Parquet file: None where the chunk has no filter, else {'offset', 'length', 'header'
    (the BloomFilterHeader fields), 'bitset_offset', 'bitset'}.  The header must say BLOCK / XXHASH / UNCOMPRESSED,
    and numBytes must fill the bloom_filter_length (when the footer has one)."""
    n = struct.unpack_from("<I", file_bytes, len(file_bytes) - 8)[0]
    fmd, end = read_struct(file_bytes, len(file_bytes) - 8 - n)
    assert end == len(file_bytes) - 8
    out = []
    for rg in fmd.get(4, []):
        row = []
        for cc in rg[1]:
            md = cc[3]
            if 14 not in md:
                assert 15 not in md
                row.append(None)
                continue
            off = md[14]
            hdr, bits_at = read_struct(file_bytes, off)
            assert hdr[2] == {1: {}} and hdr[3] == {1: {}} and hdr[4] == {1: {}}, hdr
            if 15 in md:
                assert md[15] == bits_at - off + hdr[1], (md[15], bits_at - off, hdr[1])
            row.append(dict(offset=off, length=md.get(15), header=hdr, bitset_offset=bits_at,
                            bitset=bytes(file_bytes[bits_at:bits_at + hdr[1]])))
        out.append(row)
    return out
