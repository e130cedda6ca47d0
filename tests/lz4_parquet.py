"""Parquet codec 5 (LZ4, Hadoop framing) as parquet-mr writes it for Paimon's 'lz4'.

  lz4_hadoop      Hadoop Lz4Codec framing of a page body's writes (blocks of chunks of raw LZ4 blocks)
  to_hadoop_lz4   an uncompressed Parquet file (pyarrow's, or parquet_pages' hand-built one) -> the same file with
                  every page body recompressed (a V1 page's definition levels and values as two writes, so two blocks;
                  a V2 page's values only; index pages stay as they are); page headers and footer are rewritten through
                  a generic Thrift compact reader / writer, CRCs are recomputed and every offset moves with the bytes

pyarrow itself writes codec 7 (LZ4_RAW) for 'lz4'."""
import struct
import zlib

import pyarrow as pa

SNAPPY, LZ4 = 1, 5

# Hadoop's BlockCompressorStream cuts a write into chunks of at most bufferSize - (bufferSize / 255 + 16) bytes;
# io.compression.codec.lz4.buffersize defaults to 256 KiB
HADOOP_LZ4_CHUNK = 262144 - (262144 // 255 + 16)


def lz4_hadoop(*writes: bytes, chunk: int = HADOOP_LZ4_CHUNK) -> bytes:
    """Hadoop Lz4Codec framing (Parquet codec 5): one block per non-empty write, [u32 BE length] then chunks of at most
    `chunk` bytes, each [u32 BE compressed length][raw LZ4 block]."""
    out = bytearray()
    for w in writes:
        if not w:
            continue
        out += struct.pack(">I", len(w))
        for c0 in range(0, len(w), chunk):
            blk = pa.compress(w[c0:c0 + chunk], codec="lz4_raw", asbytes=True)
            out += struct.pack(">I", len(blk)) + blk
    return bytes(out)


def _compress(codec: int, *writes: bytes) -> bytes:
    """The writes of one page body under `codec`; only Hadoop's LZ4 framing shows where one write ends."""
    if codec == LZ4:
        return lz4_hadoop(*writes)
    return pa.compress(b"".join(writes), codec={SNAPPY: "snappy"}[codec], asbytes=True)

# Thrift compact types
_T, _F, _BYTE, _I16, _I32, _I64, _DOUBLE, _BINARY, _LIST, _SET, _MAP, _STRUCT = range(1, 13)


def _varint(b, p):
    v = sh = 0
    while True:
        x = b[p]
        p += 1
        v |= (x & 0x7F) << sh
        sh += 7
        if not x & 0x80:
            return v, p


def _zz(v):
    return (v >> 1) ^ -(v & 1)


def _uvar(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _enc_zz(v):
    return _uvar((v << 1) ^ (v >> 63))


def _read(b, p, t):
    if t in (_T, _F):
        return t == _T, p
    if t == _BYTE:
        return b[p], p + 1
    if t in (_I16, _I32, _I64):
        v, p = _varint(b, p)
        return _zz(v), p
    if t == _DOUBLE:
        return bytes(b[p:p + 8]), p + 8
    if t == _BINARY:
        n, p = _varint(b, p)
        return bytes(b[p:p + n]), p + n
    if t in (_LIST, _SET):
        h = b[p]
        p += 1
        n, et = h >> 4, h & 15
        if n == 15:
            n, p = _varint(b, p)
        items = []
        for _ in range(n):
            if et in (_T, _F):                          # a bool element is one byte
                v, p = b[p], p + 1
            else:
                v, p = _read(b, p, et)
            items.append(v)
        return (et, items), p
    if t == _MAP:
        n, p = _varint(b, p)
        if n == 0:
            return (0, 0, []), p
        kv = b[p]
        p += 1
        items = []
        for _ in range(n):
            k, p = _read(b, p, kv >> 4)
            v, p = _read(b, p, kv & 15)
            items.append((k, v))
        return (kv >> 4, kv & 15, items), p
    if t == _STRUCT:
        return read_struct(b, p)
    raise ValueError(f"thrift type {t}")


def read_struct(b, p=0):
    """-> ({field id: [type, value]}, end)"""
    fields, last = {}, 0
    while True:
        h = b[p]
        p += 1
        if h == 0:
            return fields, p
        t, d = h & 15, h >> 4
        if d:
            fid = last + d
        else:
            v, p = _varint(b, p)
            fid = _zz(v)
        last = fid
        val, p = _read(b, p, t)
        fields[fid] = [t, val]


def _write(t, v):
    if t in (_I16, _I32, _I64):
        return _enc_zz(v)
    if t == _BYTE:
        return bytes([v & 255])
    if t == _DOUBLE:
        return v
    if t == _BINARY:
        return _uvar(len(v)) + v
    if t in (_LIST, _SET):
        et, items = v
        out = bytearray([(len(items) << 4) | et] if len(items) < 15 else [0xF0 | et]) + (_uvar(len(items)) if len(items) >= 15 else b"")
        for x in items:
            out += bytes([x]) if et in (_T, _F) else _write(et, x)
        return bytes(out)
    if t == _MAP:
        kt, vt, items = v
        if not items:
            return b"\x00"
        return _uvar(len(items)) + bytes([(kt << 4) | vt]) + b"".join(_write(kt, k) + _write(vt, x) for k, x in items)
    if t == _STRUCT:
        return write_struct(v)
    raise ValueError(f"thrift type {t}")


def write_struct(fields) -> bytes:
    out, last = bytearray(), 0
    for fid in sorted(fields):
        t, v = fields[fid]
        wt = (_T if v else _F) if t in (_T, _F) else t
        d = fid - last
        out += bytes([(d << 4) | wt]) if 0 < d <= 15 else bytes([wt]) + _enc_zz(fid)
        if t not in (_T, _F):
            out += _write(t, v)
        last = fid
    return bytes(out + b"\x00")


def to_hadoop_lz4(data: bytes, codec: int = LZ4, raw_first_v2: bool = False) -> bytes:
    """An uncompressed Parquet file -> the same file with codec 5 pages (`codec` = SNAPPY: Snappy pages over the same
    page bodies).  raw_first_v2: the first V2 data page of every chunk keeps its values uncompressed and says so
    (is_compressed = false), as a writer may under any codec."""
    assert data[:4] == b"PAR1" and data[-4:] == b"PAR1"
    (flen,) = struct.unpack("<I", data[-8:-4])
    meta, _ = read_struct(data, len(data) - 8 - flen)
    leaves = meta[2][1][1][1:]                          # schema elements after the root (flat files)
    optional = [e[3][1] == 1 for e in leaves]
    out = bytearray(b"PAR1")
    for rg in meta[4][1][1]:
        rg_start, rg_comp = None, 0
        for ci, cc in enumerate(rg[1][1][1]):
            md = cc[3][1]
            assert md[4][1] == 0, "the source file must be uncompressed"
            old0 = min(md[f][1] for f in (9, 11) if f in md)
            pos, end = old0, old0 + md[7][1]
            new0, moved, v2_seen = len(out), {}, False
            while pos < end:
                hdr, body0 = read_struct(data, pos)
                body = data[body0:body0 + hdr[3][1]]
                moved[pos] = len(out)
                kind = hdr[1][1]
                if kind == 1:                            # index pages: skipped by readers, left as they are
                    stored = body
                elif kind == 3:                          # V2: levels stay, values are compressed
                    v2 = hdr[8][1]
                    lv = v2[5][1] + v2.get(6, [0, 0])[1]
                    raw = raw_first_v2 and not v2_seen
                    stored = body if raw else body[:lv] + _compress(codec, body[lv:])
                    v2[7] = [_F, False] if raw else [_T, True]
                    v2_seen = True
                elif kind == 0 and optional[ci]:        # V1: levels and values are two writes
                    n_def = 4 + struct.unpack("<I", body[:4])[0]
                    stored = _compress(codec, body[:n_def], body[n_def:])
                else:
                    stored = _compress(codec, body)
                hdr[3][1] = len(stored)
                if 4 in hdr:                             # the CRC covers the stored bytes
                    hdr[4][1] = struct.unpack("<i", struct.pack("<I", zlib.crc32(stored)))[0]
                out += write_struct(hdr) + stored
                pos = body0 + len(body)
            md[4][1] = codec
            md[7][1] = len(out) - new0
            for f in (9, 10, 11):
                if f in md:
                    md[f][1] = moved[md[f][1]]
            if 2 in cc and cc[2][1]:                     # (pyarrow writes 0)
                cc[2][1] = new0
            rg_start = new0 if rg_start is None else rg_start
            rg_comp += len(out) - new0
        if 5 in rg:
            rg[5][1] = rg_start
        if 6 in rg:
            rg[6][1] = rg_comp
    footer = write_struct(meta)
    return bytes(out + footer + struct.pack("<I", len(footer)) + b"PAR1")
