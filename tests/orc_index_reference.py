"""A plain numpy model of the ORC row index and bloom filters the encoder writes with a row index stride, and a
protobuf reader of the index sections, independent of the library's orc_meta.cc and orc_encode.cu.

The rules restate the public ORC v1 specification ("Row Group Index", "Bloom Filter Index") and orc-core's
BloomFilter / Murmur3 (the writer Paimon's ORC format uses):
  * row groups of `stride` rows counted from each stripe's first row, the last one of a stripe short;
  * per row group and column the statistics orc_stats_reference.column_stats gives its rows; the root's
    numberOfValues = the row group's rows;
  * per stream of a column, in stream order, the position of the row group's first value: PRESENT [offset, 0, 0],
    BYTE DATA and integer RLE streams [offset, 0], BOOLEAN DATA [offset, 0, bit], FLOAT / DOUBLE / string / DECIMAL
    DATA [offset]; with compression the offset of the chunk header comes first;
  * a BLOOM_FILTER_UTF8 filter per row group of num_bits = nb + 64 - nb % 64 bits, nb = (int)(-stride ln fpp /
    (ln 2)^2), and k = max(1, round(num_bits / stride ln 2)) hash functions: integers and DATE through Thomas Wang's
    64-bit hash (Java's arithmetic >>), FLOAT widened to double and DOUBLE by their IEEE bits (NaN canonical) through
    the same hash, strings and BINARY through Murmur3 hash64 with seed 104729; bit i (1..k) of a hash is
    h1 + i * h2 in wrapping 32-bit arithmetic, its bits flipped when negative, modulo num_bits.
"""
import math
import struct

import numpy as np

import orc_stats_reference as ref
from orc_stats_reference import BINARY, BOOLEAN, DATE, DECIMAL, STRING, VARCHAR

M64 = (1 << 64) - 1
SEED = 104729
C1, C2 = 0x87c37b91114253d5, 0x4cf5ad432745937f
BYTES_KINDS = (STRING, VARCHAR, BINARY)
PRESENT, DATA, LENGTH, SECONDARY, ROW_INDEX, BLOOM_FILTER_UTF8 = 0, 1, 2, 5, 6, 8


# ---- hashes and filters


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def _fmix(h):
    h ^= h >> 33
    h = (h * 0xff51afd7ed558ccd) & M64
    h ^= h >> 33
    h = (h * 0xc4ceb9fe1a85ec53) & M64
    return h ^ (h >> 33)


def murmur3_hash64(data: bytes, seed: int = SEED) -> int:
    h, n = seed, len(data) // 8
    for i in range(n):
        k = struct.unpack_from("<Q", data, 8 * i)[0]
        h ^= (_rotl((k * C1) & M64, 31) * C2) & M64
        h = (_rotl(h, 27) * 5 + 0x52dce729) & M64
    tail = data[8 * n:]
    if tail:
        k = int.from_bytes(tail, "little")
        h ^= (_rotl((k * C1) & M64, 31) * C2) & M64
    return _fmix(h ^ len(data))


def wang64(keys) -> np.ndarray:
    """Thomas Wang's 64-bit hash of int64 keys, with Java's arithmetic >>"""
    k = np.asarray(keys, np.int64).view(np.uint64).copy()
    u = np.uint64

    def sar(x, r):
        return (x.view(np.int64) >> np.int64(r)).view(np.uint64)
    with np.errstate(over="ignore"):
        k = ~k + (k << u(21))
        k ^= sar(k, 24)
        k = k + (k << u(3)) + (k << u(8))
        k ^= sar(k, 14)
        k = k + (k << u(2)) + (k << u(4))
        k ^= sar(k, 28)
        k = k + (k << u(31))
    return k


def double_bits(values) -> np.ndarray:
    d = np.asarray(values, np.float64)
    bits = d.view(np.int64).copy()
    bits[np.isnan(d)] = 0x7ff8000000000000
    return bits


def hashes(kind, values, valid) -> np.ndarray:
    """the 64-bit hashes of the non-null values of a column, as uint64"""
    valid = np.asarray(valid, bool)
    if kind in BYTES_KINDS:
        return np.array([murmur3_hash64(bytes(v)) for v, ok in zip(values, valid) if ok], np.uint64)
    v = np.asarray(values)[valid]
    if kind in ref.FLOAT_KINDS:
        return wang64(double_bits(v.astype(np.float64)))
    assert kind not in (BOOLEAN, DECIMAL), kind
    return wang64(v.astype(np.int64))


def sizing(entries: int, fpp: float):
    """(num_bits, k) of orc-core's BloomFilter(entries, fpp)"""
    nb = int(-entries * math.log(fpp) / (math.log(2) ** 2))
    bits = nb + 64 - nb % 64
    return bits, max(1, int(math.floor(bits / entries * math.log(2) + 0.5)))


def bloom_bitset(h: np.ndarray, num_bits: int, k: int) -> bytes:
    """the filter of hashes h as little-endian 64-bit words"""
    words = np.zeros(num_bits // 64, np.uint64)
    h = np.asarray(h, np.uint64)
    h1 = (h & np.uint64(0xffffffff)).astype(np.uint32)
    h2 = (h >> np.uint64(32)).astype(np.uint32)
    with np.errstate(over="ignore"):
        for i in range(1, k + 1):
            c = h1 + np.uint32(i) * h2
            c = np.where(c & np.uint32(0x80000000), ~c, c)
            p = (c % np.uint32(num_bits)).astype(np.uint64)
            np.bitwise_or.at(words, p >> np.uint64(6), np.uint64(1) << (p & np.uint64(63)))
    return words.astype("<u8").tobytes()


# ---- row groups, statistics, position counts


def row_groups(n_rows: int, stripe_rows: int, stride: int):
    """per stripe, the [r0, r1) of its row groups (rows of the file)"""
    stripe_rows = (stripe_rows + 7) & ~7
    return [[(r0, min(g0 + stripe_rows, n_rows, r0 + stride)) for r0 in range(g0, min(g0 + stripe_rows, n_rows), stride)]
            for g0 in range(0, n_rows, stripe_rows)]


def expected_entries(columns, n_rows, stripe_rows, stride):
    """columns: [(kind, values, valid, scale)] -> per stripe, per column (root first), the statistics of each row
    group"""
    out = []
    for groups in row_groups(n_rows, stripe_rows, stride):
        cols = [[{"values": r1 - r0, "has_null": False} for r0, r1 in groups]]
        for kind, values, valid, scale in columns:
            cols.append([ref.column_stats(kind, values[r0:r1], np.asarray(valid)[r0:r1], scale) for r0, r1 in groups])
        out.append(cols)
    return out


def data_positions(kind: int) -> int:
    """positions of the DATA stream of a column of `kind` without compression"""
    if kind == BOOLEAN:
        return 3
    if kind in (ref.FLOAT_KINDS + BYTES_KINDS + (DECIMAL,)):
        return 1
    return 2


def position_count(kind: int, has_present: bool, compressed: bool) -> int:
    """the positions of an entry of a column: its PRESENT (when the stripe has one), DATA and LENGTH / SECONDARY"""
    streams = [3] if has_present else []
    streams.append(data_positions(kind))
    if kind in BYTES_KINDS + (DECIMAL,):
        streams.append(2)
    return sum(streams) + (len(streams) if compressed else 0)


# ---- reading a file's index sections


def uvarints(b: bytes):
    out, p = [], 0
    while p < len(b):
        v, p = ref._varint(b, p)
        out.append(v)
    return out


def inflate(section: bytes, codec: int, decompress=None) -> bytes:
    """a section of a file of compression `codec` (0 NONE, 5 ZSTD): its chunks inflated by decompress(frame)"""
    if codec == 0:
        return bytes(section)
    out, p = bytearray(), 0
    while p < len(section):
        h = section[p] | section[p + 1] << 8 | section[p + 2] << 16
        n = h >> 1
        body = bytes(section[p + 3:p + 3 + n])
        out += body if h & 1 else decompress(body)
        p += 3 + n
    return bytes(out)


class Stripe:
    def __init__(self):
        self.rows = 0
        self.index_length = 0
        self.index = {}           # column -> [(positions, statistics)] per row group
        self.bloom = {}           # column -> [(k, bit set bytes)] per row group
        self.streams = {}         # (column, kind) -> the stored bytes
        self.order = []           # (kind, column) of every stream in file order


def read_file(blob: bytes, decompress=None):
    """(row index stride, [Stripe]) of an ORC file; decompress(frame) inflates a ZSTD chunk"""
    ps_len = blob[-1]
    ps = {f: v for f, _, v in ref.fields(blob[-1 - ps_len:-1])}
    codec = ps.get(2, 0)
    foot_end = len(blob) - 1 - ps_len
    footer = ref.fields(inflate(blob[foot_end - ps[1]:foot_end], codec, decompress))
    stride = next((v for f, _, v in footer if f == 8), 0)
    out = []
    for f, _, si in footer:
        if f != 3:
            continue
        info = {g: v for g, _, v in ref.fields(si)}
        st = Stripe()
        st.rows, st.index_length = info[5], info.get(2, 0)
        off = info[1]
        foot_at = off + info.get(2, 0) + info[3]
        sf = ref.fields(inflate(blob[foot_at:foot_at + info[4]], codec, decompress))
        pos = off
        for g, _, s in sf:
            if g != 1:
                continue
            d = {h: v for h, _, v in ref.fields(s)}
            kind, col, n = d.get(1, 0), d.get(2, 0), d.get(3, 0)
            stored = blob[pos:pos + n]
            st.order.append((kind, col))
            if kind == ROW_INDEX:
                st.index[col] = [(uvarints(next((v for h, _, v in e if h == 1), b"")),
                                  ref.parse_column_statistics(next(v for h, _, v in e if h == 2)))
                                 for e in (ref.fields(x) for h, _, x in ref.fields(inflate(stored, codec, decompress)))]
            elif kind == BLOOM_FILTER_UTF8:
                st.bloom[col] = [({h: v for h, _, v in ref.fields(x)}[1], {h: v for h, _, v in ref.fields(x)}[3])
                                 for _, _, x in ref.fields(inflate(stored, codec, decompress))]
            else:
                st.streams[(col, kind)] = stored
            pos += n
        out.append(st)
    return stride, out
