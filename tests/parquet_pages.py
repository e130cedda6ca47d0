"""Parquet files built page by page on the host, for tests that need byte layouts no writer produces on request.

Written from the public Parquet format specification (parquet.thrift, Encodings.md) and the Thrift compact protocol;
independent of the repository's encoder, so it can judge the decoder.  The pieces:

  ThriftWriter         compact protocol: i32 / i64 / binary / bool / list / struct, short- and long-form field headers
  plain / hybrid /     value encoders: PLAIN for every physical type, the RLE / bit-packed hybrid from an explicit run
  delta_binary_packed  plan, DELTA_BINARY_PACKED with a free block shape, forced and garbage miniblock widths
  data_page_v1 / v2,   pages, each with optional CRC, page Statistics, unknown header fields and (V2) is_compressed
  dictionary_page,
  index_page
  kv_file              a flat KeyValue-shaped file ([_KEY_pk, _SEQUENCE_NUMBER, _VALUE_KIND, pk, value columns...]) of
                       row groups whose value chunks are lists of pages; returns the file bytes

Expected values are plain Python values (None = NULL); they are the reference the decoder is compared with.
"""
import struct
import zlib
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np
import pyarrow as pa

# parquet.thrift enums
BOOLEAN, INT32, INT64, FLOAT, DOUBLE, BYTE_ARRAY = 0, 1, 2, 4, 5, 6
E_PLAIN, E_PLAIN_DICTIONARY, E_RLE, E_DELTA_BINARY_PACKED, E_RLE_DICTIONARY = 0, 2, 3, 5, 8
UNCOMPRESSED, SNAPPY, GZIP, ZSTD = 0, 1, 2, 6
DATA_PAGE, INDEX_PAGE, DICTIONARY_PAGE, DATA_PAGE_V2 = 0, 1, 2, 3
REQUIRED, OPTIONAL = 0, 1
# ConvertedType
UTF8, DATE, INT_8, INT_16 = 0, 6, 15, 16
_CODEC_NAME = {SNAPPY: "snappy", GZIP: "gzip", ZSTD: "zstd"}

# Thrift compact protocol wire types
CT_TRUE, CT_FALSE, CT_BYTE, CT_I16, CT_I32, CT_I64, CT_DOUBLE, CT_BINARY, CT_LIST, CT_SET, CT_MAP, CT_STRUCT = range(1, 13)


def uvarint(v: int) -> bytes:
    assert v >= 0
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def zigzag(v: int) -> int:
    return (v << 1) ^ (v >> 63) if v < 0 else v << 1


class ThriftWriter:
    """Thrift compact protocol.  A field header is short-form (id delta 1..15 in the high nibble) unless the delta is
    out of range or `long_form` is asked for: then the type byte is followed by the zigzag varint of the id."""

    def __init__(self):
        self.b = bytearray()
        self._last = [0]

    def field(self, fid: int, ttype: int, long_form: bool = False):
        d = fid - self._last[-1]
        if 0 < d <= 15 and not long_form:
            self.b.append((d << 4) | ttype)
        else:
            self.b.append(ttype)
            self.b += uvarint(zigzag(fid))
        self._last[-1] = fid

    def i32(self, fid, v, long_form=False):
        self.field(fid, CT_I32, long_form)
        self.b += uvarint(zigzag(v))

    def i64(self, fid, v, long_form=False):
        self.field(fid, CT_I64, long_form)
        self.b += uvarint(zigzag(v))

    def i16(self, fid, v, long_form=False):
        self.field(fid, CT_I16, long_form)
        self.b += uvarint(zigzag(v))

    def byte(self, fid, v, long_form=False):
        self.field(fid, CT_BYTE, long_form)
        self.b.append(v & 0xFF)

    def double(self, fid, v, long_form=False):
        self.field(fid, CT_DOUBLE, long_form)
        self.b += struct.pack("<d", v)

    def binary(self, fid, v: bytes, long_form=False):
        self.field(fid, CT_BINARY, long_form)
        self.b += uvarint(len(v)) + bytes(v)

    def bool(self, fid, v: bool, long_form=False):
        self.field(fid, CT_TRUE if v else CT_FALSE, long_form)       # the value lives in the field header

    def list_begin(self, fid, elem_type, n, ttype=CT_LIST, long_form=False):
        self.field(fid, ttype, long_form)
        self.b += bytes([(n << 4) | elem_type]) if n < 15 else bytes([0xF0 | elem_type]) + uvarint(n)

    def list_i32(self, fid, vals, long_form=False):
        self.list_begin(fid, CT_I32, len(vals), long_form=long_form)
        for v in vals:
            self.b += uvarint(zigzag(v))

    def list_binary(self, fid, vals, long_form=False):
        self.list_begin(fid, CT_BINARY, len(vals), long_form=long_form)
        for v in vals:
            self.b += uvarint(len(v)) + bytes(v)

    def struct_begin(self, fid, long_form=False):
        self.field(fid, CT_STRUCT, long_form)
        self._last.append(0)

    def elem_begin(self):                              # a struct that is a list element
        self._last.append(0)

    def struct_end(self):
        self.b.append(0)
        self._last.pop()

    def stop(self) -> bytes:
        self.b.append(0)
        return bytes(self.b)


def unknown_fields(w: ThriftWriter):
    """Fields no parquet.thrift version defines, one of every Thrift type, all with long-form ids: readers must skip
    them."""
    w.bool(100, True, long_form=True)
    w.bool(101, False, long_form=True)
    w.byte(102, -5, long_form=True)
    w.i16(103, -1234, long_form=True)
    w.i32(1000, 1 << 30, long_form=True)
    w.i64(1001, -(1 << 62), long_form=True)
    w.double(1002, 2.5, long_form=True)
    w.binary(1003, b"\x00unknown\xff" * 3, long_form=True)
    w.list_binary(1004, [b"a", b"", b"x" * 200] + [b"%d" % i for i in range(20)], long_form=True)
    w.list_begin(1005, CT_I32, 3, ttype=CT_SET, long_form=True)
    for v in (7, -8, 1 << 20):
        w.b += uvarint(zigzag(v))
    w.list_begin(1006, CT_TRUE, 3, long_form=True)     # booleans inside a container take one byte each
    w.b += bytes([1, 2, 1])
    w.field(1007, CT_MAP, long_form=True)              # an empty map: size 0, no key / value types
    w.b.append(0)
    w.struct_begin(30000, long_form=True)              # a nested struct with a struct, a list and a bool inside
    w.i32(1, 9)
    w.struct_begin(2)
    w.binary(1, b"inner")
    w.bool(2, True)
    w.struct_end()
    w.list_binary(3, [b"p", b"q"])
    w.i64(40, 1 << 40, long_form=True)
    w.struct_end()


# ------------------------------------------------------------------ value encoders

def pack_bits(values, width: int) -> bytes:
    """LSB-first bit packing of unsigned values (the hybrid's bit-packed runs, DELTA miniblocks)."""
    v = np.asarray(values, dtype=np.uint64)
    if width == 0 or v.size == 0:
        return b""
    bits = ((v[:, None] >> np.arange(width, dtype=np.uint64)) & np.uint64(1)).astype(np.uint8)
    return np.packbits(bits.ravel(), bitorder="little").tobytes()


def plain(phys: int, values: Sequence) -> bytes:
    """PLAIN values of the non-null cells.  FLOAT / DOUBLE values may be given as floats or as bit patterns (ints)."""
    if phys == BOOLEAN:
        return np.packbits(np.asarray(values, dtype=np.uint8), bitorder="little").tobytes()
    if phys == BYTE_ARRAY:
        return b"".join(struct.pack("<I", len(v)) + bytes(v) for v in values)
    if phys in (FLOAT, DOUBLE):
        fmt, ifmt = ("<f", "<I") if phys == FLOAT else ("<d", "<Q")
        return b"".join(struct.pack(ifmt, v) if isinstance(v, int) else struct.pack(fmt, v) for v in values)
    return np.asarray(values, dtype=np.int32 if phys == INT32 else np.int64).astype("<i8" if phys == INT64 else "<i4").tobytes()


def hybrid(width: int, plan) -> bytes:
    """The RLE / bit-packed hybrid stream of an explicit run plan: ("rle", count, value) and ("packed", values).  A
    packed run holds whole groups of 8; only the last run of a stream may be padded (with zeros)."""
    out = bytearray()
    for i, run in enumerate(plan):
        if run[0] == "rle":
            _, n, v = run
            out += uvarint(n << 1) + int(v).to_bytes((width + 7) // 8, "little")
        else:
            vals = list(run[1])
            assert i == len(plan) - 1 or len(vals) % 8 == 0, "a padded bit-packed run must end the stream"
            groups = (len(vals) + 7) // 8
            vals += [0] * (8 * groups - len(vals))
            out += uvarint((groups << 1) | 1) + pack_bits(vals, width)
    return bytes(out)


def plan_values(plan) -> List[int]:
    out = []
    for run in plan:
        out += [run[2]] * run[1] if run[0] == "rle" else list(run[1])
    return out


def delta_binary_packed(values: Sequence[int], bits: int, block: int = 128, minis: int = 4, widths=None,
                        garbage=None) -> bytes:
    """DELTA_BINARY_PACKED of `values` (ints of a `bits`-bit type; deltas wrap like the type's arithmetic).
    `widths`: a miniblock bit width per miniblock index (cycled), used where it is at least the width the deltas need.
    `garbage`: bit widths written for the unneeded miniblocks of the last block (the spec lets them be anything; no
    data follows them)."""
    assert block % 128 == 0 and block % minis == 0 and (block // minis) % 32 == 0
    mask = (1 << bits) - 1

    def signed(x):
        x &= mask
        return x - (1 << bits) if x >> (bits - 1) else x

    vals = [signed(v) for v in values]
    out = bytearray(uvarint(block) + uvarint(minis) + uvarint(len(vals)) + uvarint(zigzag(vals[0] if vals else 0)))
    mini = block // minis
    deltas = [signed(vals[i] - vals[i - 1]) for i in range(1, len(vals))]
    for b0 in range(0, len(deltas), block):
        blk = deltas[b0:b0 + block]
        mn = min(blk)
        out += uvarint(zigzag(mn))
        rel = [d - mn for d in blk]                    # 0 <= rel < 2^bits
        used = (len(blk) + mini - 1) // mini
        ws = []
        for m in range(minis):
            if m < used:
                w = max(rel[m * mini:(m + 1) * mini]).bit_length()
                if widths is not None:
                    f = widths[((b0 // block) * minis + m) % len(widths)]
                    w = max(w, f)
                ws.append(w)
            else:
                ws.append(garbage[m % len(garbage)] if garbage else 0)
        out += bytes(ws)
        for m in range(used):
            chunk = rel[m * mini:(m + 1) * mini]
            chunk += [0] * (mini - len(chunk))         # the last miniblock is padded to its full size
            out += pack_bits(np.array(chunk, dtype=np.uint64), ws[m])
    return bytes(out)


# ------------------------------------------------------------------ pages

@dataclass
class Page:
    data: bytes            # header + body as stored
    kind: int              # page type
    encoding: int
    num_values: int        # data pages: rows (flat columns); dictionary pages: entries
    unc: int               # uncompressed page size (header excluded)
    comp: int              # stored page size (header excluded)


def _compress(codec: int, body: bytes) -> bytes:
    if codec == UNCOMPRESSED:
        return body
    return pa.compress(body, codec=_CODEC_NAME[codec], asbytes=True)


def _header(kind, unc, comp, stored: bytes, crc: bool, extras: bool, sub_id: int, sub) -> bytes:
    w = ThriftWriter()
    w.i32(1, kind)
    w.i32(2, unc)
    w.i32(3, comp)
    if crc:
        w.i32(4, struct.unpack("<i", struct.pack("<I", zlib.crc32(stored)))[0])
    w.struct_begin(sub_id)
    sub(w)
    w.struct_end()
    if extras:
        unknown_fields(w)
    return w.stop()


def _statistics(w: ThriftWriter, fid: int, null_count: int, lo: bytes, hi: bytes):
    w.struct_begin(fid)
    w.binary(1, hi)
    w.binary(2, lo)
    w.i64(3, null_count)
    w.i64(4, 2)
    w.binary(5, hi)
    w.binary(6, lo)
    w.bool(7, True)
    w.bool(8, True)
    w.struct_end()


def levels(valid: Sequence[bool], plan=None) -> bytes:
    """Definition levels of a flat OPTIONAL column (bit width 1): one bit-packed run, or an explicit plan."""
    if plan is None:
        plan = [("packed", [1 if v else 0 for v in valid])] if len(valid) else []
    assert plan_values(plan)[:len(valid)] == [1 if v else 0 for v in valid]
    return hybrid(1, plan)


def data_page_v1(num_values: int, values: bytes, encoding: int, defs: Optional[bytes] = None, codec=UNCOMPRESSED,
                 crc=False, stats=False, extras=False, null_count=0) -> Page:
    """V1: body = [definition levels: 4-byte length + hybrid stream (OPTIONAL columns)] [values], compressed whole."""
    body = (struct.pack("<I", len(defs)) + defs if defs is not None else b"") + values
    stored = _compress(codec, body)

    def sub(w):
        w.i32(1, num_values)
        w.i32(2, encoding)
        w.i32(3, E_RLE)
        w.i32(4, E_RLE)
        if stats:
            _statistics(w, 5, null_count, b"\x00" * 4, b"\x7f" * 4)
    return Page(_header(DATA_PAGE, len(body), len(stored), stored, crc, extras, 5, sub) + stored, DATA_PAGE, encoding,
                num_values, len(body), len(stored))


def data_page_v2(num_values: int, values: bytes, encoding: int, defs: bytes = b"", null_count=0, codec=UNCOMPRESSED,
                 is_compressed: Optional[bool] = None, crc=False, stats=False, extras=False) -> Page:
    """V2: body = [definition levels, no length word, never compressed] [values, compressed unless is_compressed is
    false].  is_compressed=None leaves the field out (it defaults to true)."""
    comp_vals = values if is_compressed is False else _compress(codec, values)
    stored = defs + comp_vals

    def sub(w):
        w.i32(1, num_values)
        w.i32(2, null_count)
        w.i32(3, num_values)
        w.i32(4, encoding)
        w.i32(5, len(defs))
        w.i32(6, 0)
        if is_compressed is not None:
            w.bool(7, is_compressed)
        if stats:
            _statistics(w, 8, null_count, b"\x00" * 4, b"\x7f" * 4)
    unc = len(defs) + len(values)
    return Page(_header(DATA_PAGE_V2, unc, len(stored), stored, crc, extras, 8, sub) + stored, DATA_PAGE_V2, encoding,
                num_values, unc, len(stored))


def dictionary_page(num_values: int, body: bytes, codec=UNCOMPRESSED, encoding=E_PLAIN, crc=False, extras=False) -> Page:
    stored = _compress(codec, body)

    def sub(w):
        w.i32(1, num_values)
        w.i32(2, encoding)
    return Page(_header(DICTIONARY_PAGE, len(body), len(stored), stored, crc, extras, 7, sub) + stored, DICTIONARY_PAGE,
                encoding, num_values, len(body), len(stored))


def index_page(body: bytes = b"index page bytes") -> Page:
    return Page(_header(INDEX_PAGE, len(body), len(body), body, False, False, 6, lambda w: None) + body, INDEX_PAGE, -1,
                0, len(body), len(body))


# ------------------------------------------------------------------ files

@dataclass
class ValueColumn:
    """A value column of a KeyValue file: its name, physical type, OPTIONAL or not, converted type, codec, and per row
    group the list of pages of its chunk (a dictionary page first, if any)."""
    name: str
    phys: int
    optional: bool
    chunks: List[List[Page]]
    codec: int = UNCOMPRESSED
    converted: Optional[int] = None


@dataclass
class _Chunk:
    phys: int
    codec: int
    pages: List[Page]
    num_values: int
    encodings: List[int] = field(default_factory=list)


def _plain_chunk(phys: int, values) -> _Chunk:
    p = data_page_v1(len(values), plain(phys, values), E_PLAIN)
    return _Chunk(phys, UNCOMPRESSED, [p], len(values))


def kv_file(rg_rows: Sequence[int], cols: Sequence[ValueColumn], key0: int = 0) -> bytes:
    """A flat KeyValue file [_KEY_pk BIGINT, _SEQUENCE_NUMBER BIGINT, _VALUE_KIND TINYINT, pk BIGINT, cols...] whose
    row groups have rg_rows rows.  pk = key0 + row (PLAIN), _SEQUENCE_NUMBER = row, _VALUE_KIND = 0."""
    schema = [(b"_KEY_pk", INT64, REQUIRED, None), (b"_SEQUENCE_NUMBER", INT64, REQUIRED, None),
              (b"_VALUE_KIND", INT32, REQUIRED, INT_8), (b"pk", INT64, REQUIRED, None)]
    schema += [(c.name.encode(), c.phys, OPTIONAL if c.optional else REQUIRED, c.converted) for c in cols]
    out = bytearray(b"PAR1")
    groups = []                                        # per row group: rows, [(offset, dict offset, chunk)]
    row = 0
    for g, n in enumerate(rg_rows):
        keys = list(range(key0 + row, key0 + row + n))
        chunks = [_plain_chunk(INT64, keys), _plain_chunk(INT64, list(range(row, row + n))),
                  _plain_chunk(INT32, [0] * n), _plain_chunk(INT64, keys)]
        for c in cols:
            pages = c.chunks[g]
            nv = sum(p.num_values for p in pages if p.kind in (DATA_PAGE, DATA_PAGE_V2))
            assert nv == n, f"column {c.name} row group {g}: pages hold {nv} rows, the row group {n}"
            chunks.append(_Chunk(c.phys, c.codec, pages, n))
        placed = []
        for ch in chunks:
            start = len(out)
            dict_off = start if ch.pages and ch.pages[0].kind == DICTIONARY_PAGE else None
            data_off = start
            for p in ch.pages:
                if p.kind in (DATA_PAGE, DATA_PAGE_V2) and data_off == start and dict_off is not None:
                    data_off = len(out)
                out += p.data
            encs = sorted({E_RLE} | {p.encoding for p in ch.pages if p.kind != INDEX_PAGE})
            unc = sum(len(p.data) - p.comp + p.unc for p in ch.pages)
            placed.append((start, data_off, dict_off, len(out) - start, unc, ch, encs))
        groups.append((n, placed))
        row += n
    w = ThriftWriter()
    w.i32(1, 1)
    w.list_begin(2, CT_STRUCT, len(schema) + 1)
    w.elem_begin()
    w.binary(4, b"schema")
    w.i32(5, len(schema))
    w.struct_end()
    for name, phys, rep, conv in schema:
        w.elem_begin()
        w.i32(1, phys)
        w.i32(3, rep)
        w.binary(4, name)
        if conv is not None:
            w.i32(6, conv)
        w.struct_end()
    w.i64(3, row)
    w.list_begin(4, CT_STRUCT, len(groups))
    for n, placed in groups:
        w.elem_begin()
        w.list_begin(1, CT_STRUCT, len(placed))
        for (start, data_off, dict_off, comp, unc, ch, encs), (name, *_rest) in zip(placed, schema):
            w.elem_begin()
            w.i64(2, start)
            w.struct_begin(3)
            w.i32(1, ch.phys)
            w.list_i32(2, encs)
            w.list_binary(3, [name])
            w.i32(4, ch.codec)
            w.i64(5, ch.num_values)
            w.i64(6, unc)
            w.i64(7, comp)
            w.i64(9, data_off)
            if dict_off is not None:
                w.i64(11, dict_off)
            w.struct_end()
            w.struct_end()
        w.i64(2, sum(p[4] for p in placed))
        w.i64(3, n)
        w.struct_end()
    w.binary(6, b"parquet_pages test builder")
    footer = w.stop()
    out += footer + struct.pack("<I", len(footer)) + b"PAR1"
    return bytes(out)



# ------------------------------------------------------------------ cases
#
# A case is the files of one sorted run and the values the value column "v" must decode to.  Floats are compared by
# bit pattern, so their expected values are the IEEE bit patterns (ints); strings and binaries are bytes.

@dataclass
class Case:
    name: str
    files: List[bytes]
    vtype: str                      # Paimon type of "v" in the read schema
    expected: list                  # values of "v" over the run, None = NULL
    pyarrow: bool = True            # pyarrow reads the files (False: a layout the spec allows and pyarrow refuses)
    crc: bool = False               # the pages carry CRCs
    data_pages: Optional[int] = None
    dict_pages: Optional[int] = None


# Paimon type -> (physical type, converted type, dictionary / value generator over an index array, bit-pattern width)
def _mix(i, mult, bits):
    return (np.asarray(i, dtype=np.uint64) * np.uint64(mult) + np.uint64(0x1234567)) & np.uint64((1 << bits) - 1)


def _signed(u, bits):
    return u.astype(np.uint32).view(np.int32) if bits == 32 else u.astype(np.uint64).view(np.int64)


def _gen_int32(i):
    v = _signed(_mix(i, 2654435761, 32), 32)
    v[: 2] = [-(1 << 31), (1 << 31) - 1][: len(v[:2])]
    return v.tolist()


def _gen_int64(i):
    v = _signed(_mix(i, 0x9E3779B97F4A7C15, 64), 64)
    v[: 2] = [-(1 << 63), (1 << 63) - 1][: len(v[:2])]
    return v.tolist()


_F32_EDGES = [0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x7FC00001, 0xFFC12345, 0x7F7FFFFF, 0x3F800000]
_F64_EDGES = [0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 0x1, 0x7FF8000000000001,
              0xFFF8123456789ABC, 0x7FEFFFFFFFFFFFFF, 0x3FF0000000000000]


def _gen_f32_bits(i, finite=False):
    v = _mix(i, 2246822519, 32)
    v[: len(_F32_EDGES)] = _F32_EDGES[: len(v)]
    if finite:                                         # no NaN / infinity (the FLOAT -> DOUBLE cast case)
        v = np.where((v & np.uint64(0x7F800000)) == np.uint64(0x7F800000), v & np.uint64(0xBFFFFFFF), v)
    return v.tolist()


def _gen_f64_bits(i):
    v = _mix(i, 0xC2B2AE3D27D4EB4F, 64)
    v[: len(_F64_EDGES)] = _F64_EDGES[: len(v)]
    return v.tolist()


def _gen_bytes(i, text):
    out = []
    for k in np.asarray(i).tolist():
        s = b"%x" % (k * 2654435761 & 0xFFFFFFFF)
        s = s * (k % 4) if k % 11 else b""
        out.append(s if text else bytes([k & 255, 0, 255]) + s)
    return out


def _f32_to_f64_bits(b):
    return np.array(b, dtype=np.uint32).view(np.float32).astype(np.float64).view(np.uint64).tolist()


# vtype -> (physical, converted, values of indices i)
FIXED_TYPES = {
    "TINYINT": (INT32, INT_8, lambda i: ((np.asarray(i) * 37 % 256) - 128).tolist()),
    "SMALLINT": (INT32, INT_16, lambda i: ((np.asarray(i) * 7919 % 65536) - 32768).tolist()),
    "INT": (INT32, None, _gen_int32),
    "DATE": (INT32, DATE, lambda i: (np.asarray(i, np.int64) * 3 - 719_528).tolist()),
    "BIGINT": (INT64, None, _gen_int64),
    "FLOAT": (FLOAT, None, _gen_f32_bits),
    "DOUBLE": (DOUBLE, None, _gen_f64_bits),
    "STRING": (BYTE_ARRAY, UTF8, lambda i: _gen_bytes(i, True)),
    "BINARY": (BYTE_ARRAY, None, lambda i: _gen_bytes(i, False)),
}
# schema evolution: the file holds INT32 / FLOAT, the table reads BIGINT / DOUBLE
CAST_TYPES = {
    "INT->BIGINT": ("BIGINT", INT32, None, _gen_int32, lambda v: v),
    "FLOAT->DOUBLE": ("DOUBLE", FLOAT, None, lambda i: _gen_f32_bits(i, finite=True), _f32_to_f64_bits),
}


def id_plan(shape: str, n: int, top: int, rng: np.random.Generator, start: int = 0):
    """A hybrid run plan of at least n values in [0, top]: only RLE runs, only bit-packed runs (the last one padded),
    or RLE runs of 1..32 values alternating with bit-packed runs, so the packed runs start at every residue mod 8 and
    every bit of a 32-bit word."""
    plan, got, k = [], 0, start

    def rand(m):
        v = rng.integers(0, top + 1, m).tolist()
        if m:
            v[m // 2] = top
        return v

    while got < n:
        if shape == "rle":
            m = [1, 2, 3, 7, 8, 9, 31, 33, 64, 100, 127, 128][k % 12]
            plan.append(("rle", m, [top, 0, top // 2, 1 if top else 0][k % 4] if k % 5 else int(rng.integers(0, top + 1))))
        elif shape == "packed":
            m = 8 * [1, 2, 3, 64, 5, 70][k % 6]
            plan.append(("packed", rand(m)))
        else:
            m = k % 32 + 1
            plan.append(("rle", m, int(rng.integers(0, top + 1))))
            if got + m < n:
                plan.append(("packed", rand(8 * (1 + k % 3))))
                m += plan[-1][1].__len__()
        got += m
        k += 1
    if plan[-1][0] == "packed" and got > n:                 # the last packed run ends with padding
        extra = min(got - n, 7)
        plan[-1] = ("packed", plan[-1][1][: len(plan[-1][1]) - extra])
    return plan


def long_plan(top: int):
    """Run headers of 3 varint bytes: an RLE run of 9000 values and a bit-packed run of 8192 groups."""
    rng = np.random.default_rng(top)
    return [("rle", 9000, top), ("packed", rng.integers(0, top + 1, 65536).tolist())]


def _dict_sizes():
    sizes = [1, 2]
    for k in range(1, 20):
        sizes += [s for s in (1 << k, (1 << k) + 1) if s not in sizes]
    return sizes


def dictionary_case(vtype: str) -> Case:
    """Dictionary-encoded pages of one column: a row group per dictionary size (1, 2, 2^k, 2^k + 1 up to 2^19 + 1, so
    widths 0 to 20 are needed); in each, pages at the needed width, one wider and 32, each with an RLE-only, a
    bit-packed-only and an alternating id stream (the alternating pages with NULLs); PLAIN_DICTIONARY and
    RLE_DICTIONARY ids in turn; a few row groups also carry a page of 3-byte run headers."""
    if vtype in CAST_TYPES:
        read_type, phys, conv, gen, to_read = CAST_TYPES[vtype]
    else:
        phys, conv, gen = FIXED_TYPES[vtype]
        read_type, to_read = vtype, (lambda v: v)
    rng = np.random.default_rng(len(vtype))
    chunks, rows, expected = [], [], []
    n_data = n_dict = 0
    for g, size in enumerate(_dict_sizes()):
        entries = gen(np.arange(size))
        read_entries = to_read(entries) if phys == FLOAT else entries
        need = (size - 1).bit_length()
        enc = E_PLAIN_DICTIONARY if g % 2 == 0 else E_RLE_DICTIONARY
        pages = [dictionary_page(size, plain(phys, entries), encoding=E_PLAIN_DICTIONARY if g % 2 == 0 else E_PLAIN)]
        n_rows = 0
        widths = sorted({need, min(need + 1, 32), 32})
        shapes = [(s, w) for w in widths for s in ("rle", "packed", "mixed")]
        if g in (0, 1, 9, len(_dict_sizes()) - 1):
            shapes.append(("long", need))
        for j, (shape, w) in enumerate(shapes):
            n = 100 + 37 * j if shape != "long" else 9000 + 65536
            plan = long_plan(size - 1) if shape == "long" else id_plan(shape, n if shape != "mixed" else (2 * n) // 3 + 1, size - 1, rng, start=j)
            valid = [True] * n if shape != "mixed" else [r % 3 != 1 for r in range(n)]
            nnz = sum(valid)
            ids = plan_values(plan)[:nnz]
            assert len(ids) == nnz
            stream = bytes([w]) + hybrid(w, plan)
            defs = levels(valid, [("rle", n, 1)] if all(valid) else None)
            if j % 2:
                pages.append(data_page_v2(n, stream, enc, defs=defs, null_count=n - nnz))
            else:
                pages.append(data_page_v1(n, stream, enc, defs=defs))
            it = iter(ids)
            expected += [read_entries[next(it)] if v else None for v in valid]
            n_rows += n
        chunks.append(pages)
        rows.append(n_rows)
        n_data += len(pages) - 1
        n_dict += 1
    col = ValueColumn("v", phys, True, chunks, converted=conv)
    return Case(f"dict_{vtype}", [kv_file(rows, [col])], read_type, expected, data_pages=n_data + 4 * len(rows),
                dict_pages=n_dict)


def rle_boolean_case() -> Case:
    """BOOLEAN cannot be dictionary-encoded; its RLE pages run the same stream shapes at width 1 (V1 and V2)."""
    rng = np.random.default_rng(1)
    pages, expected = [], []
    shapes = ["rle", "packed", "mixed", "long"] * 2
    for j, shape in enumerate(shapes):
        n = 300 + 41 * j if shape != "long" else 9000 + 65536
        valid = [True] * n if shape in ("rle", "long") else [r % 4 != 2 for r in range(n)]
        nnz = sum(valid)
        plan = long_plan(1) if shape == "long" else id_plan(shape, nnz, 1, rng, start=j)
        vals = plan_values(plan)[:nnz]
        stream = hybrid(1, plan)
        body = struct.pack("<I", len(stream)) + stream
        defs = levels(valid, [("rle", n, 1)] if all(valid) else None)
        if j >= 4:
            pages.append(data_page_v2(n, body, E_RLE, defs=defs, null_count=n - nnz))
        else:
            pages.append(data_page_v1(n, body, E_RLE, defs=defs))
        it = iter(vals)
        expected += [bool(next(it)) if v else None for v in valid]
    rows = sum(p.num_values for p in pages)
    return Case("rle_boolean", [kv_file([rows], [ValueColumn("v", BOOLEAN, True, [pages])])], "BOOLEAN", expected,
                data_pages=len(pages) + 4)


def _def_pages(sizes, rng, v2_every=2, shapes=("rle", "packed", "mixed")):
    """PLAIN BIGINT pages whose definition levels take the given run shapes at width 1."""
    pages, expected = [], []
    for j, n in enumerate(sizes):
        shape = shapes[j % len(shapes)]
        plan = id_plan(shape, n, 1, rng, start=j)
        bits = plan_values(plan)[:n]
        vals = _gen_int64(np.arange(j * 1000, j * 1000 + sum(bits)))
        defs = hybrid(1, plan)
        if j % v2_every == v2_every - 1:
            pages.append(data_page_v2(n, plain(INT64, vals), E_PLAIN, defs=defs, null_count=n - sum(bits)))
        else:
            pages.append(data_page_v1(n, plain(INT64, vals), E_PLAIN, defs=defs))
        it = iter(vals)
        expected += [next(it) if b else None for b in bits]
    return pages, expected


def definition_levels_case() -> Case:
    """Definition levels of every run shape, V1 and V2, including runs with 2- and 3-byte headers."""
    rng = np.random.default_rng(2)
    pages, expected = _def_pages([100, 517, 1000, 64, 9001, 8191, 30000, 77, 3], rng)
    lp = long_plan(1)
    n = len(plan_values(lp))
    bits = plan_values(lp)
    vals = _gen_int64(np.arange(sum(bits)))
    pages.append(data_page_v1(n, plain(INT64, vals), E_PLAIN, defs=hybrid(1, lp)))
    it = iter(vals)
    expected += [next(it) if b else None for b in bits]
    rows = sum(p.num_values for p in pages)
    return Case("def_levels", [kv_file([rows], [ValueColumn("v", INT64, True, [pages])])], "BIGINT", expected,
                data_pages=len(pages) + 4)


SMALL_PAGES = [1, 7, 31, 32, 33, 63]


def small_pages_file(seed: int, cycles: int, key0: int = 0):
    """Pages of 1, 7, 31, 32, 33 and 63 rows in turn: a cycle is 167 rows (7 mod 32), so over 32 cycles the page starts
    fall on every bit of a validity word and several pages OR into one word."""
    rng = np.random.default_rng(seed)
    pages, expected = _def_pages(SMALL_PAGES * cycles, rng, v2_every=3)
    rows = sum(p.num_values for p in pages)
    return kv_file([rows], [ValueColumn("v", INT64, True, [pages])], key0=key0), expected, len(pages)


def small_pages_case() -> Case:
    f, expected, n = small_pages_file(3, 32)
    return Case("small_pages", [f], "BIGINT", expected, data_pages=n + 4)


def small_pages_run_case() -> Case:
    """A run of several such files: every file after the first starts at a row that is not a multiple of 32."""
    files, expected, n_pages, key0 = [], [], 0, 0
    for i, cycles in enumerate([1, 3, 2, 5]):
        f, e, n = small_pages_file(10 + i, cycles, key0=key0)
        files.append(f)
        expected += e
        key0 += len(e)
        n_pages += n + 4
    return Case("small_pages_run", files, "BIGINT", expected, data_pages=n_pages)


DELTA_SHAPES = [(128, 4), (128, 1), (256, 8), (512, 4)]


def _delta_values(kind: str, n: int, bits: int, rng) -> List[int]:
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    if n == 0:
        return []
    if kind == "extremes":                             # the type's edges: every delta wraps
        return [[lo, hi, 0, hi, lo, -1][i % 6] for i in range(n)]
    if kind == "random":                               # deltas over the full range: natural width 32 / 64
        return rng.integers(lo, hi, n, endpoint=True, dtype=np.int64 if bits == 64 else np.int32).tolist()
    if kind == "constant":                             # width 0
        return [hi - 7 * i if bits == 64 else ((hi - 7 * i - lo) % (1 << 32)) + lo for i in range(n)]
    return [int(x) for x in np.cumsum(rng.integers(-3, 4, n)) + (hi - 100)]   # small deltas, widths forced wider


def delta_case(vtype: str) -> Case:
    """DELTA_BINARY_PACKED pages: block / miniblock shapes 128/4, 128/1, 256/8, 512/4; miniblock widths 0, 1, 31, 32 (and
    33, 63, 64 on INT64); first values at the type's extremes and wrapping deltas; totals of 0, 1, one short of a
    miniblock and exact block multiples; garbage widths for the unneeded miniblocks of the last block."""
    bits = 32 if vtype == "INT" else 64
    phys = INT32 if bits == 32 else INT64
    rng = np.random.default_rng(bits)
    forced = [1, 31, 32] + ([33, 63, 64] if bits == 64 else [])
    pages, expected = [], []
    j = 0
    for block, minis in DELTA_SHAPES:
        mini = block // minis
        for kind in ("extremes", "random", "constant", "forced"):
            for total in (0, 1, mini - 1, 2 * block + 1, mini + 5):
                with_nulls = (j % 3 == 1) or total == 0
                n = total + (total // 3 + 4 if with_nulls else 0)
                valid = [True] * n
                if with_nulls:
                    nulls = set(rng.choice(n, n - total, replace=False).tolist())
                    valid = [r not in nulls for r in range(n)]
                vals = _delta_values(kind, total, bits, rng)
                body = delta_binary_packed(vals, bits, block, minis, widths=forced if kind == "forced" else None,
                                           garbage=[255, 7, 200, 65, 0, 3, 99, 64] if j % 2 else None)
                defs = levels(valid)
                if j % 2:
                    pages.append(data_page_v2(n, body, E_DELTA_BINARY_PACKED, defs=defs, null_count=n - total))
                else:
                    pages.append(data_page_v1(n, body, E_DELTA_BINARY_PACKED, defs=defs))
                it = iter(vals)
                expected += [next(it) if v else None for v in valid]
                j += 1
    rows = sum(p.num_values for p in pages)
    return Case(f"delta_{vtype}", [kv_file([rows], [ValueColumn("v", phys, True, [pages])])], vtype, expected,
                data_pages=len(pages) + 4)


def headers_case(codec: int) -> Case:
    """Page headers with CRCs, page Statistics and unknown fields of every Thrift type (long-form ids, a list of
    binaries, a nested struct); an index page between data pages; a dictionary page compressed under the codec; V2 pages
    with is_compressed = false (and true) under it; a PLAIN fallback page behind the dictionary."""
    rng = np.random.default_rng(codec)
    entries = _gen_bytes(np.arange(300), True)
    pages = [dictionary_page(300, plain(BYTE_ARRAY, entries), codec=codec, crc=True, extras=True), index_page()]
    expected = []

    def dict_ids(n, valid):
        nnz = sum(valid)
        plan = id_plan("mixed", nnz, 299, rng)
        return plan_values(plan)[:nnz], bytes([9]) + hybrid(9, plan)

    for j in range(6):
        n = 150 + 13 * j
        valid = [r % 5 != 3 for r in range(n)]
        nnz = sum(valid)
        if j == 4:                                     # PLAIN fallback
            vals = _gen_bytes(np.arange(1000 + nnz * j, 1000 + nnz * (j + 1)), True)
            body, enc = plain(BYTE_ARRAY, vals), E_PLAIN
        else:
            ids, body = dict_ids(n, valid)
            vals, enc = [entries[i] for i in ids], E_RLE_DICTIONARY
        defs = levels(valid)
        if j % 2:
            pages.append(data_page_v2(n, body, enc, defs=defs, null_count=n - nnz, codec=codec,
                                      is_compressed=(j != 1) if codec != UNCOMPRESSED else None, crc=True,
                                      stats=True, extras=True))
        else:
            pages.append(data_page_v1(n, body, enc, defs=defs, codec=codec, crc=True, stats=True, extras=True,
                                      null_count=n - nnz))
        if j == 2:
            pages.append(index_page(b"between data pages"))
        it = iter(vals)
        expected += [next(it) if v else None for v in valid]
    rows = sum(p.num_values for p in pages if p.kind in (DATA_PAGE, DATA_PAGE_V2))
    col = ValueColumn("v", BYTE_ARRAY, True, [pages], codec=codec, converted=UTF8)
    name = {UNCOMPRESSED: "none", SNAPPY: "snappy", GZIP: "gzip", ZSTD: "zstd"}[codec]
    return Case(f"headers_{name}", [kv_file([rows], [col])], "STRING", expected, crc=True, data_pages=6 + 4,
                dict_pages=1)


def well_formed_cases():
    """name -> builder of every well-formed case."""
    cases = {f"dict_{t}": (lambda t=t: dictionary_case(t)) for t in list(FIXED_TYPES) + list(CAST_TYPES)}
    cases["rle_boolean"] = rle_boolean_case
    cases["def_levels"] = definition_levels_case
    cases["small_pages"] = small_pages_case
    cases["small_pages_run"] = small_pages_run_case
    cases["delta_INT"] = lambda: delta_case("INT")
    cases["delta_BIGINT"] = lambda: delta_case("BIGINT")
    for c, nm in ((UNCOMPRESSED, "none"), (SNAPPY, "snappy"), (GZIP, "gzip"), (ZSTD, "zstd")):
        cases[f"headers_{nm}"] = lambda c=c: headers_case(c)
    return cases


# ------------------------------------------------------------------ malformed streams
#
# Each returns (file bytes, vtype).  Every wrong read a decoder that does not check these could make stays inside the
# file or the decoder's own buffers, except where noted.

def _one_page_file(phys, conv, page, dict_page=None):
    pages = ([dict_page] if dict_page else []) + [page]
    return kv_file([page.num_values], [ValueColumn("v", phys, True, [pages], converted=conv)])


def _short_ids(phys, conv, vtype):
    """A dictionary-id stream that covers 60 of the page's 100 non-null values."""
    n = 100
    entries = FIXED_TYPES[vtype][2](np.arange(16))
    page = data_page_v1(n, bytes([4]) + hybrid(4, [("rle", 60, 3)]), E_RLE_DICTIONARY, defs=levels([True] * n))
    return _one_page_file(phys, conv, page, dictionary_page(16, plain(phys, entries))), vtype


def _truncated_ids():
    """A dictionary-id stream whose bit-packed run (10 groups of 8 ids at width 4: 40 bytes) has lost its last 5."""
    n = 100
    stream = bytes([4]) + hybrid(4, [("rle", 20, 1), ("packed", [i % 16 for i in range(80)])])
    page = data_page_v1(n, stream[:-5], E_RLE_DICTIONARY, defs=levels([True] * n))
    return _one_page_file(INT32, None, page, dictionary_page(16, plain(INT32, _gen_int32(np.arange(16))))), "INT"


def _short_booleans():
    """RLE booleans: the stream covers 40 of 100 values."""
    stream = hybrid(1, [("rle", 40, 1)])
    page = data_page_v1(100, struct.pack("<I", len(stream)) + stream, E_RLE, defs=levels([True] * 100))
    return _one_page_file(BOOLEAN, None, page), "BOOLEAN"


def _short_defs():
    """PLAIN BIGINT, 100 values present, but the definition levels cover 50 rows."""
    page = data_page_v1(100, plain(INT64, list(range(100))), E_PLAIN, defs=hybrid(1, [("rle", 50, 1)]))
    return _one_page_file(INT64, None, page), "BIGINT"


def _truncated_defs():
    """PLAIN BIGINT, 100 values present; the definition levels' bit-packed run (13 groups) keeps 6 of its 13 bytes."""
    defs = hybrid(1, [("packed", [1] * 104)])
    page = data_page_v1(100, plain(INT64, list(range(100))), E_PLAIN, defs=defs[:1 + 6])
    return _one_page_file(INT64, None, page), "BIGINT"


def _dictionary_overclaims():
    """An INT32 dictionary page that claims 20 entries with the bytes of 10 (40 bytes); ids reach 19.  The chunk is
    uncompressed and the data page that follows is longer than the 40 missing bytes, so reading the missing entries
    lands in that page."""
    n = 100
    ids = [i % 20 for i in range(n)]
    page = data_page_v1(n, bytes([5]) + hybrid(5, [("packed", ids)]), E_RLE_DICTIONARY, defs=levels([True] * n))
    assert len(page.data) > 40
    return _one_page_file(INT32, None, page, dictionary_page(20, plain(INT32, list(range(1000, 1010))))), "INT"


def malformed_cases():
    """name -> builder of (file bytes, vtype) for each malformed stream the decoder must refuse."""
    return {
        "ids_stream_short_int": lambda: _short_ids(INT32, None, "INT"),
        "ids_stream_short_string": lambda: _short_ids(BYTE_ARRAY, UTF8, "STRING"),
        "ids_run_truncated": _truncated_ids,
        "bool_stream_short": _short_booleans,
        "def_stream_short": _short_defs,
        "def_run_truncated": _truncated_defs,
        "dict_page_overclaims": _dictionary_overclaims,
    }


# ------------------------------------------------------------------ comparison in the expected values' terms

def _float_bits(vtype: str):
    return {"FLOAT": np.uint32, "DOUBLE": np.uint64}.get(vtype)


def arrow_values(arr, vtype: str) -> list:
    """A pyarrow array of "v" as expected values: floats as bit patterns, strings as bytes."""
    arr = arr.combine_chunks() if hasattr(arr, "combine_chunks") else arr
    if pa.types.is_date32(arr.type):                   # (days outside Python's date range)
        arr = arr.cast(pa.int32())
    valid = arr.is_valid().to_numpy(zero_copy_only=False)
    ub = _float_bits(vtype)
    if ub is not None:
        vals = np.asarray(arr.fill_null(0).to_numpy(zero_copy_only=False)).view(ub).tolist()
    else:
        vals = [v.encode() if isinstance(v, str) else v for v in arr.to_pylist()]
    return [v if ok else None for v, ok in zip(vals, valid)]


def column_values(col, vtype: str) -> list:
    """A decoded paimon_b200 Column as expected values (its validity bit by bit, floats as bit patterns)."""
    from paimon_b200.columnar import unpack_validity
    n = len(col)
    valid = unpack_validity(col.valid, n)
    ub = _float_bits(vtype)
    if ub is not None:
        vals = np.asarray(col.data[:n]).view(ub).tolist()
    elif vtype == "BOOLEAN":
        vals = [bool(x) for x in np.asarray(col.data[:n]).tolist()]
    elif vtype in ("STRING", "BINARY"):
        raw, offs = np.asarray(col.data).tobytes(), np.asarray(col.offsets)
        vals = [raw[offs[i]:offs[i + 1]] for i in range(n)]
    else:
        vals = np.asarray(col.data[:n]).tolist()
    return [v if ok else None for v, ok in zip(vals, valid)]


def first_mismatch(got: list, want: list) -> str:
    if len(got) != len(want):
        return f"{len(got)} values, expected {len(want)}"
    for i, (a, b) in enumerate(zip(got, want)):
        if a != b:
            return f"row {i}: {a!r} != {b!r}"
    return "equal"
