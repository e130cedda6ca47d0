"""An independent model of Paimon's bloom-filter file index, restated from the Java sources, for the tests of
file_index.py, xxhash64_device.cuh and k_bloom_build:
  FastHash (paimon-common/.../fileindex/bloomfilter/FastHash.java): Thomas Wang's 64-bit hash (Java's arithmetic >>)
    of integers and of Float.floatToIntBits / Double.doubleToLongBits; XXH64 with seed 0 of bytes
    (LongHashFunction.xx()), restated here from the published specification in pure Python;
  BloomFilter64 (paimon-common/.../utils/BloomFilter64.java): sizing, addHash, testHash;
  BloomFilterFileIndex.Writer.serializedBytes: big-endian hash function count, then the bit set;
  FileIndexFormat.Writer / Reader (paimon-common/.../fileindex/FileIndexFormat.java);
  the bucket order of a java.util.HashMap of column names (DataFileIndexWriter.serializeMaintainers).
No library code is imported."""
import math
import struct

import numpy as np

M64 = (1 << 64) - 1
P1, P2, P3, P4, P5 = (0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63,
                      0x27D4EB2F165667C5)


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def _round(acc, lane):
    return _rotl((acc + lane * P2) & M64, 31) * P1 & M64


def xxh64(data: bytes) -> int:
    """XXH64(data, seed 0) as an unsigned 64-bit integer."""
    n, i = len(data), 0
    if n >= 32:
        v = [(P1 + P2) & M64, P2, 0, (-P1) & M64]
        while n - i >= 32:
            for j in range(4):
                v[j] = _round(v[j], int.from_bytes(data[i + 8 * j:i + 8 * j + 8], "little"))
            i += 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & M64
        for x in v:
            h = ((h ^ _round(0, x)) * P1 + P4) & M64
    else:
        h = P5
    h = (h + n) & M64
    while n - i >= 8:
        h = (_rotl(h ^ _round(0, int.from_bytes(data[i:i + 8], "little")), 27) * P1 + P4) & M64
        i += 8
    if n - i >= 4:
        h = (_rotl(h ^ (int.from_bytes(data[i:i + 4], "little") * P1 & M64), 23) * P2 + P3) & M64
        i += 4
    while i < n:
        h = _rotl(h ^ (data[i] * P5 & M64), 11) * P1 & M64
        i += 1
    h ^= h >> 33
    h = h * P2 & M64
    h ^= h >> 29
    h = h * P3 & M64
    h ^= h >> 32
    return h


def s64(x: int) -> int:
    x &= M64
    return x - (1 << 64) if x >> 63 else x


def s32(x: int) -> int:
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x >> 31 else x


def get_long_hash(key: int) -> int:
    """FastHash.getLongHash on a Java long (Python's >> on a signed int is Java's arithmetic >>)."""
    key = s64(~key + (key << 21))
    key = s64(key ^ (key >> 24))
    key = s64(key + (key << 3) + (key << 8))
    key = s64(key ^ (key >> 14))
    key = s64(key + (key << 2) + (key << 4))
    key = s64(key ^ (key >> 28))
    return s64(key + (key << 31))


def float_to_int_bits(bits32: int) -> int:
    """Float.floatToIntBits of the float with these raw bits, as a signed int."""
    if (bits32 >> 23) & 0xFF == 0xFF and bits32 & 0x7FFFFF:
        bits32 = 0x7FC00000
    return s32(bits32)


def double_to_long_bits(bits64: int) -> int:
    if (bits64 >> 52) & 0x7FF == 0x7FF and bits64 & ((1 << 52) - 1):
        bits64 = 0x7FF8000000000000
    return s64(bits64)


INTEGER_ROOTS = {"TINYINT", "SMALLINT", "INT", "INTEGER", "BIGINT", "DATE", "TIME", "TIMESTAMP"}
BYTES_ROOTS = {"CHAR", "VARCHAR", "STRING", "BINARY", "VARBINARY", "BYTES"}


def fast_hash(logical: str, value) -> int:
    """The 64-bit hash of one non-null value of a Paimon type.  Integers (and the stored INT32 / INT64 of DATE, TIME
    and TIMESTAMP: millis for p <= 3, micros above) are Python ints; FLOAT / DOUBLE are Python floats or
    ('bits', raw bits) for NaN payloads; strings are str (their UTF-8 bytes) or bytes."""
    root = logical.upper().split("(")[0].strip()
    if root in INTEGER_ROOTS:
        return get_long_hash(int(value))
    if root == "FLOAT":
        bits = value[1] if isinstance(value, tuple) else int(np.float32(value).view(np.uint32))
        return get_long_hash(float_to_int_bits(bits))
    if root == "DOUBLE":
        bits = value[1] if isinstance(value, tuple) else int(np.float64(value).view(np.uint64))
        return get_long_hash(double_to_long_bits(bits))
    if root in BYTES_ROOTS:
        return s64(xxh64(value.encode("utf-8") if isinstance(value, str) else bytes(value)))
    if root == "BOOLEAN":
        raise ValueError("Does not support type boolean")
    if root == "DECIMAL":
        raise ValueError("Does not support decimal")
    raise ValueError(logical)


def java_int_cast(x: float) -> int:
    """(int) of a double: NaN -> 0, saturating, toward zero."""
    if x != x:
        return 0
    return max(-(1 << 31), min((1 << 31) - 1, int(x)))


def sizing(items: int, fpp: float):
    """BloomFilter64(items, fpp): (numBits, numHashFunctions), or None where the Java int arithmetic overflows and the
    bit set cannot be allocated."""
    nb = java_int_cast(-items * math.log(fpp) / (math.log(2) * math.log(2)))     # >= 0 for items > 0, fpp < 1
    num_bits = s32(nb + (8 - nb % 8))
    if num_bits <= 0:
        return None
    k = max(1, java_int_cast(math.floor(num_bits / items * math.log(2) + 0.5)))
    return num_bits, k


def positions(hash64: int, k: int, num_bits: int):
    """BloomFilter64.addHash's bit positions."""
    h1, h2 = s32(hash64), s32((hash64 & M64) >> 32)
    out = []
    for i in range(1, k + 1):
        c = s32(h1 + i * h2)
        if c < 0:
            c = ~c
        out.append(c % num_bits)
    return out


class BloomFilter:
    def __init__(self, items: int = 1_000_000, fpp: float = 0.1):
        self.num_bits, self.k = sizing(items, fpp)
        self.bits = bytearray(self.num_bits // 8)

    @staticmethod
    def from_bytes(data: bytes) -> "BloomFilter":
        f = BloomFilter.__new__(BloomFilter)
        f.k = struct.unpack(">i", data[:4])[0]
        f.bits = bytearray(data[4:])
        f.num_bits = len(f.bits) * 8
        return f

    def add_hash(self, h: int) -> None:
        for p in positions(h, self.k, self.num_bits):
            self.bits[p >> 3] |= 1 << (p & 7)

    def test_hash(self, h: int) -> bool:
        return all(self.bits[p >> 3] >> (p & 7) & 1 for p in positions(h, self.k, self.num_bits))

    def serialized(self) -> bytes:
        return struct.pack(">i", self.k) + bytes(self.bits)


def filter_of(logical: str, values, items: int = 1_000_000, fpp: float = 0.1) -> bytes:
    """BloomFilterFileIndex.Writer over `values` (None = NULL, skipped), serialized."""
    f = BloomFilter(items, fpp)
    for v in values:
        if v is not None:
            f.add_hash(fast_hash(logical, v))
    return f.serialized()


def java_utf(s: str) -> bytes:
    """DataOutputStream.writeUTF."""
    b = bytearray()
    for ch in s:
        cp = ord(ch)
        units = [cp] if cp < 0x10000 else [0xD800 + ((cp - 0x10000) >> 10), 0xDC00 + ((cp - 0x10000) & 0x3FF)]
        for u in units:
            if 1 <= u <= 0x7F:
                b.append(u)
            elif u <= 0x7FF:
                b += bytes([0xC0 | (u >> 6), 0x80 | (u & 0x3F)])
            else:
                b += bytes([0xE0 | (u >> 12), 0x80 | ((u >> 6) & 0x3F), 0x80 | (u & 0x3F)])
    return struct.pack(">H", len(b)) + bytes(b)


def container(columns) -> bytes:
    """FileIndexFormat.Writer.writeColumnIndexes over [(column, [(index type, bytes)])] in that order."""
    names = sum(len(java_utf(c)) + sum(len(java_utf(t)) for t, _ in ts) for c, ts in columns)
    head_len = 8 + 4 + 4 + 4 + 8 * sum(len(ts) for _, ts in columns) + 4 * len(columns) + 4 + names
    head = struct.pack(">qiii", 1493475289347502, 1, head_len, len(columns))
    body = b""
    for c, ts in columns:
        head += java_utf(c) + struct.pack(">i", len(ts))
        for t, data in ts:
            head += java_utf(t) + struct.pack(">ii", head_len + len(body), len(data))
            body += data
    return head + struct.pack(">i", 0) + body


def read_container(data: bytes):
    """FileIndexFormat.Reader: [(column, {index type: bytes})] in the order of the head."""
    def utf(pos):                        # DataInputStream.readUTF: modified UTF-8 -> UTF-16 units -> str
        (n,) = struct.unpack_from(">H", data, pos)
        b, i, units = data[pos + 2:pos + 2 + n], 0, []
        while i < len(b):
            if b[i] < 0x80:
                units.append(b[i])
                i += 1
            elif b[i] < 0xE0:
                units.append((b[i] & 0x1F) << 6 | b[i + 1] & 0x3F)
                i += 2
            else:
                units.append((b[i] & 0x0F) << 12 | (b[i + 1] & 0x3F) << 6 | b[i + 2] & 0x3F)
                i += 3
        text = b"".join(struct.pack(">H", u) for u in units).decode("utf-16-be", "surrogatepass")
        return text, pos + 2 + n
    magic, version, head_len, n_cols = struct.unpack_from(">qiii", data, 0)
    assert magic == 1493475289347502 and version == 1
    pos, out = 20, []
    for _ in range(n_cols):
        col, pos = utf(pos)
        (n_idx,) = struct.unpack_from(">i", data, pos)
        pos += 4
        idx = {}
        for _ in range(n_idx):
            t, pos = utf(pos)
            start, length = struct.unpack_from(">ii", data, pos)
            pos += 8
            idx[t] = data[start:start + length]
        out.append((col, idx))
    assert struct.unpack_from(">i", data, pos)[0] == 0 and pos + 4 == head_len
    return out


def java_hash(s: str) -> int:
    h = 0
    for ch in s:
        cp = ord(ch)
        for u in ([cp] if cp < 0x10000 else [0xD800 + ((cp - 0x10000) >> 10), 0xDC00 + ((cp - 0x10000) & 0x3FF)]):
            h = (31 * h + u) & 0xFFFFFFFF
    return h


def hashmap_buckets(names):
    """The buckets, in iteration order, of a HashMap filled with `names` by computeIfAbsent (which resizes before an
    insert once the map holds more than 3/4 of its table), each bucket as a set: the order of names inside one bucket
    depends on insertion history, the order of the buckets does not."""
    cap = 16
    for size in range(len(names)):          # the table seen by the (size + 1)-th insert
        if size > cap * 3 // 4:
            cap *= 2
    buckets = {}
    for n in names:
        h = java_hash(n)
        buckets.setdefault((h ^ (h >> 16)) & (cap - 1), set()).add(n)
    return [buckets[b] for b in sorted(buckets)]
