"""Streams for the page decompressors and the reference libraries' readings of them, shared by the host tests
(test_codecs_cpu.py) and the device tests (test_gpu_codecs.py).

- zstd frames from libzstd (through pyarrow) that between them hold multi-block frames, raw and RLE blocks, raw, RLE,
  1- and 4-stream Huffman and treeless literals, and several frames (and a skippable frame) in one stream;
- raw DEFLATE and zlib streams from zlib under every strategy (Z_HUFFMAN_ONLY, Z_RLE, Z_FIXED, Z_FILTERED, stored
  blocks at level 0, empty stored blocks from sync flushes);
- gzip streams: concatenated members and hand-framed members with FEXTRA, FNAME, FCOMMENT and FHCRC.

The references return the bytes the library produces, or None when it refuses.  Two checks the decoders skip are
turned off in the references the way the decoders skip them: the gzip CRC32 (and header CRC16) and the zlib Adler-32
are recomputed before zlib sees the stream.
"""
import random
import struct
import zlib
from typing import Dict, Optional, Set, Tuple

import numpy as np
import pyarrow as pa

SNAPPY, ZSTD, RAW_DEFLATE, GZIP, ZLIB = 0, 1, 2, 3, 4


def sample_inputs() -> Dict[str, bytes]:
    rng = random.Random(5)
    g = np.random.default_rng(5)
    words = [b"alpha", b"beta", b"gamma", b"paimon", b"lsm", b"merge", b"tree", b"x", b"yy"]
    return {
        "text_600k": b" ".join(rng.choice(words) for _ in range(100_000)),
        "random_300k": g.integers(0, 256, 300_000, dtype=np.uint8).tobytes(),
        "zeros_400k": bytes(400_000),
        "rows_300k": b"".join(b"%08d|user_%07d|%d;" % (i % 977, i, i % 13) for i in range(14_000)),
        "small_text": b"hello paimon hello merge tree " * 6,
        "one": b"x",
        "int64_sorted": np.arange(0, 40_000, dtype=np.int64).tobytes(),
        "lowcard": g.integers(0, 7, 200_000, dtype=np.uint8).tobytes(),
        "padded_counter": b"".join(bytes(9) + b"%06d" % i for i in range(20_000)),   # RLE literals at level 19
    }


# ------------------------------------------------------------------ zstd

def zstd(data: bytes, level: int = 3) -> bytes:
    return pa.Codec("zstd", compression_level=level).compress(data, asbytes=True)


def libzstd(stream: bytes, size: int) -> Optional[bytes]:
    """libzstd at the exact size (pyarrow refuses a stream that produces fewer bytes than asked for)."""
    try:
        return pa.decompress(stream, decompressed_size=size, codec="zstd", asbytes=True)
    except OSError:
        return None


def zstd_corpus() -> Dict[str, Tuple[bytes, bytes]]:
    """name -> (stream, expected output)"""
    d = sample_inputs()
    out = {}
    for name, data in d.items():
        for level in (1, 3, 19):
            out[f"{name}_l{level}"] = (zstd(data, level), data)
    a, b = d["text_600k"][:70_000], d["rows_300k"][:90_000]
    out["three_frames"] = (zstd(a, 3) + zstd(b"", 3) + zstd(b, 19), a + b)
    skippable = struct.pack("<II", 0x184D2A53, 5) + b"skip!"
    out["skippable_then_frame"] = (skippable + zstd(b, 1), b)
    return out


def zstd_kinds(stream: bytes) -> Set[str]:
    """The block and literals-section kinds of every block of every frame (RFC 8878 3.1.1, 3.1.1.2 and 3.1.1.3.1)."""
    kinds, pos = set(), 0
    while pos < len(stream):
        magic = int.from_bytes(stream[pos:pos + 4], "little")
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            kinds.add("skippable_frame")
            pos += 8 + int.from_bytes(stream[pos + 4:pos + 8], "little")
            continue
        assert magic == 0xFD2FB528
        kinds.add("frame")
        fhd = stream[pos + 4]
        single, did, fcs = (fhd >> 5) & 1, fhd & 3, fhd >> 6
        pos += 5 + (0 if single else 1) + [0, 1, 2, 4][did] + [1 if single else 0, 2, 4, 8][fcs]
        blocks = 0
        while True:
            bh = int.from_bytes(stream[pos:pos + 3], "little")
            last, btype, bsize = bh & 1, (bh >> 1) & 3, bh >> 3
            blocks += 1
            kinds.add(["raw_block", "rle_block", "compressed_block"][btype])
            if btype == 2:
                lh = stream[pos + 3]
                lt, sf = lh & 3, (lh >> 2) & 3
                kinds.add(["raw_literals", "rle_literals", "huffman", "treeless"][lt] +
                          ("" if lt < 2 else ("_1_stream" if sf == 0 else "_4_streams")))
            pos += 3 + (1 if btype == 1 else bsize)
            if last:
                break
        if blocks > 1:
            kinds.add("multi_block_frame")
        pos += 4 if fhd & 4 else 0
    return kinds


# ------------------------------------------------------------------ DEFLATE

STRATEGIES = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman_only": zlib.Z_HUFFMAN_ONLY,
              "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}


def deflate(data: bytes, level: int = 6, strategy: int = zlib.Z_DEFAULT_STRATEGY, wbits: int = -15,
            sync_every: int = 0) -> bytes:
    co = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, strategy)
    if not sync_every:
        return co.compress(data) + co.flush()
    out = b"".join(co.compress(data[i:i + sync_every]) + co.flush(zlib.Z_SYNC_FLUSH)
                   for i in range(0, len(data), sync_every))
    return out + co.flush()


def deflate_corpus(wbits: int) -> Dict[str, Tuple[bytes, bytes]]:
    """name -> (stream, expected output); wbits -15 raw DEFLATE, 15 zlib."""
    d = sample_inputs()
    out = {}
    for name in ("text_600k", "random_300k", "zeros_400k", "rows_300k", "small_text", "one", "lowcard"):
        data = d[name]
        for sname, strat in STRATEGIES.items():
            out[f"{name}_{sname}"] = (deflate(data, 6, strat, wbits), data)
        out[f"{name}_stored"] = (deflate(data, 0, wbits=wbits), data)
    data = d["rows_300k"][:100_000]
    out["sync_flushes"] = (deflate(data, 6, wbits=wbits, sync_every=7_000), data)
    out["empty"] = (deflate(b"", 6, wbits=wbits), b"")
    return out


def _inflate_end(stream: bytes, start: int) -> Optional[Tuple[bytes, int]]:
    """zlib's raw inflate of stream[start:]: (output, end of the DEFLATE data), or None."""
    d = zlib.decompressobj(-15)
    try:
        got = d.decompress(stream[start:]) + d.flush()
    except zlib.error:
        return None
    if not d.eof:
        return None
    return got, len(stream) - len(d.unused_data)


def zlib_raw(stream: bytes) -> Optional[bytes]:
    r = _inflate_end(stream, 0)
    return None if r is None else r[0]


def zlib_zlib(stream: bytes) -> Optional[bytes]:
    """zlib's reading of a zlib stream with the Adler-32 recomputed (the decoder requires it but does not verify it)."""
    r = _inflate_end(stream, 2)
    if r is None or len(stream) - r[1] < 4:
        return None
    patched = stream[:r[1]] + struct.pack(">I", zlib.adler32(r[0])) + stream[r[1] + 4:]
    d = zlib.decompressobj(15)
    try:
        got = d.decompress(patched) + d.flush()
    except zlib.error:
        return None
    return got if d.eof else None


def _gzip_header_end(s: bytes, pos: int) -> Optional[int]:
    """Where a member's header ends (RFC 1952 2.3), found only to place the CRCs; zlib judges the header."""
    if len(s) - pos < 10:
        return None
    flg, p = s[pos + 3], pos + 10
    if flg & 4:
        if p + 2 > len(s):
            return None
        p += 2 + int.from_bytes(s[p:p + 2], "little")
    for bit in (8, 16):
        if flg & bit:
            z = s.find(b"\x00", p)
            if z < 0:
                return None
            p = z + 1
    return p + (2 if flg & 2 else 0)


def zlib_gzip(stream: bytes) -> Optional[bytes]:
    """zlib's reading of concatenated gzip members, each with its header CRC16 and CRC32 recomputed (the decoder
    skips both); the ISIZE and everything else is zlib's to check."""
    out, pos = bytearray(), 0
    while pos < len(stream):
        h = _gzip_header_end(stream, pos)
        if h is None or h > len(stream):
            return None
        r = _inflate_end(stream, h)
        if r is None or len(stream) - r[1] < 8:
            return None
        hdr = bytearray(stream[pos:h])
        if hdr[3] & 2:
            hdr[-2:] = struct.pack("<H", zlib.crc32(bytes(hdr[:-2])) & 0xFFFF)
        member = bytes(hdr) + stream[h:r[1]] + struct.pack("<I", zlib.crc32(r[0])) + stream[r[1] + 4:r[1] + 8]
        d = zlib.decompressobj(31)
        try:
            got = d.decompress(member) + d.flush()
        except zlib.error:
            return None
        if not d.eof or d.unused_data:
            return None
        out += got
        pos = r[1] + 8
    return bytes(out)


def gzip_member(data: bytes, extra: Optional[bytes] = None, name: Optional[bytes] = None,
                comment: Optional[bytes] = None, hcrc: bool = False, level: int = 6) -> bytes:
    """One gzip member framed by hand (RFC 1952), with the optional header fields asked for."""
    flg = (4 if extra is not None else 0) | (8 if name is not None else 0) | (16 if comment is not None else 0) | \
          (2 if hcrc else 0)
    hdr = bytes([0x1F, 0x8B, 8, flg]) + struct.pack("<I", 1_700_000_000) + bytes([0, 3])
    if extra is not None:
        hdr += struct.pack("<H", len(extra)) + extra
    if name is not None:
        hdr += name + b"\x00"
    if comment is not None:
        hdr += comment + b"\x00"
    if hcrc:
        hdr += struct.pack("<H", zlib.crc32(hdr) & 0xFFFF)
    return hdr + deflate(data, level) + struct.pack("<II", zlib.crc32(data), len(data) & 0xFFFFFFFF)


def gzip_corpus() -> Dict[str, Tuple[bytes, bytes]]:
    d = sample_inputs()
    a, b, c = d["text_600k"][:50_000], d["rows_300k"][:80_000], d["small_text"]
    out = {}
    for name in ("text_600k", "random_300k", "zeros_400k", "small_text", "one"):
        out[name] = (gzip_member(d[name]), d[name])
    out["empty"] = (gzip_member(b""), b"")
    out["fextra"] = (gzip_member(a, extra=b"AP\x04\x00abcd"), a)
    out["fname"] = (gzip_member(a, name=b"page.bin"), a)
    out["fcomment"] = (gzip_member(a, comment=b"a comment"), a)
    out["fhcrc"] = (gzip_member(a, hcrc=True), a)
    out["all_header_fields"] = (gzip_member(b, extra=b"", name=b"n", comment=b"", hcrc=True), b)
    out["three_members"] = (gzip_member(a) + gzip_member(b"", name=b"e") + gzip_member(b, level=1, hcrc=True), a + b)
    out["stored_member"] = (gzip_member(c, level=0) + gzip_member(c, comment=b"c"), c + c)
    return out


def pad8(data: bytes) -> bytes:
    """data padded with zeros to a multiple of 8 bytes (the values of an INT64 page)."""
    return data + bytes(-len(data) % 8)


def _with_content_size(frame: bytes, delta: int) -> bytes:
    """A zstd frame whose Frame_Content_Size field says `delta` more than it does."""
    fhd = frame[4]
    single, did, fcs = (fhd >> 5) & 1, fhd & 3, fhd >> 6
    n = [1 if single else 0, 2, 4, 8][fcs]
    assert n
    p = 5 + (0 if single else 1) + [0, 1, 2, 4][did]
    v = int.from_bytes(frame[p:p + n], "little") + delta
    return frame[:p] + v.to_bytes(n, "little") + frame[p + n:]


def malformed_streams() -> Dict[str, Tuple[int, bytes, int]]:
    """name -> (mode, stream, output size): malformed zstd and gzip streams that libzstd / zlib refuse, one per rule
    the decoders enforce.  Every size is a multiple of 8."""
    d = pad8(sample_inputs()["rows_300k"][:5000])
    z = zstd(d, 3)
    bh = 5 + (0 if (z[4] >> 5) & 1 else 1) + [0, 1, 2, 4][z[4] & 3] + [1 if (z[4] >> 5) & 1 else 0, 2, 4, 8][z[4] >> 6]
    g = gzip_member(d)
    return {
        "zstd_truncated": (ZSTD, z[:-3], len(d)),
        "zstd_content_size_above": (ZSTD, _with_content_size(z, 8), len(d)),
        "zstd_content_size_below": (ZSTD, _with_content_size(z, -8), len(d)),
        "zstd_bad_magic": (ZSTD, b"\x29" + z[1:], len(d)),
        "zstd_reserved_block_type": (ZSTD, z[:bh] + bytes([z[bh] | 6]) + z[bh + 1:], len(d)),
        "zstd_skippable_frame_past_input": (ZSTD, z + struct.pack("<II", 0x184D2A50, 100) + b"abc", len(d)),
        "zstd_output_past_size": (ZSTD, z, len(d) - 8),
        "gzip_wrong_isize": (GZIP, g[:-4] + struct.pack("<I", len(d) + 8), len(d)),
        "gzip_truncated": (GZIP, g[:-5], len(d)),
        "gzip_reserved_flag": (GZIP, g[:3] + b"\x20" + g[4:], len(d)),
        "gzip_trailing_bytes": (GZIP, g + b"\x1f\x8b", len(d)),
        "gzip_bad_stored_length": (GZIP, gzip_member(d, level=0)[:11] + b"\x00\x00" + gzip_member(d, level=0)[13:], len(d)),
        "gzip_output_past_size": (GZIP, g, len(d) - 8),
    }


def malformed_chunks() -> Dict[str, Tuple[int, bytes, int]]:
    """name -> (mode, body, output size): malformed zstd and raw DEFLATE bodies of ORC compression chunks."""
    d = sample_inputs()["rows_300k"][:1200]
    z, zl, stored = zstd(d, 3), deflate(d, 9), deflate(d, 0)
    return {
        "zstd_truncated": (ZSTD, z[:-2], len(d)),
        "zstd_content_size_above": (ZSTD, _with_content_size(z, 1), len(d)),
        "zstd_bad_magic": (ZSTD, b"\x29" + z[1:], len(d)),
        "deflate_truncated": (RAW_DEFLATE, zl[:len(zl) // 2], len(d)),
        "deflate_reserved_block_type": (RAW_DEFLATE, bytes([zl[0] | 6]) + zl[1:], len(d)),
        "deflate_bad_stored_length": (RAW_DEFLATE, stored[:1] + b"\x00\x00" + stored[3:], len(d)),
    }


def reference(mode: int, stream: bytes, size: int) -> Optional[bytes]:
    """The reference library's reading of a stream that must produce `size` bytes, or None when it refuses."""
    if mode == SNAPPY:
        from snappy_streams import libsnappy
        return libsnappy(stream, size)
    if mode == ZSTD:
        return libzstd(stream, size)
    got = {RAW_DEFLATE: zlib_raw, GZIP: zlib_gzip, ZLIB: zlib_zlib}[mode](stream)
    return got if got is not None and len(got) == size else None
