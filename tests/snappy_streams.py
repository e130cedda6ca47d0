"""A Snappy element writer, written from the public Snappy format description and independent of any compressor: a
stream is a varint preamble (the uncompressed length) followed by elements whose kind and encoding the caller picks.

- literal(data, length_bytes): 0 = the length inline in the tag (1..60), 1..4 = that many little-endian length bytes
  behind tag 60..63 (a short literal may take more length bytes than it needs);
- copy(offset, length, kind): kind 1 (length 4..11, offset < 2048), 2 (length 1..64, offset < 65536) or 4 (length
  1..64, any 32-bit offset).  A copy whose offset is below its length overlaps its own output.

Every element appends to `expected`, the bytes a decoder must produce.  pyarrow's Snappy compressor never writes
copy-4 elements or literals with 3- or 4-byte lengths, since it compresses 64 KiB fragments; these streams do.
"""
import random
import struct
from typing import Dict, Optional

import pyarrow as pa


def varint(v: int) -> bytes:
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def preamble(stream: bytes) -> Optional[int]:
    """The uncompressed length a stream declares, under libsnappy's rule (at most 5 bytes, the fifth below 16); None
    when the preamble is malformed."""
    v = 0
    for i in range(5):
        if i >= len(stream):
            return None
        b = stream[i]
        if i == 4 and b > 15:
            return None
        v |= (b & 0x7F) << (7 * i)
        if not b & 0x80:
            return v
    return None


def libsnappy(stream: bytes, size: int) -> Optional[bytes]:
    """libsnappy (through pyarrow) at the exact size: the output, or None when it refuses the stream or the stream
    declares another size (pyarrow accepts an output buffer larger than the preamble)."""
    if preamble(stream) != size:
        return None
    try:
        return pa.decompress(stream, decompressed_size=size, codec="snappy", asbytes=True)
    except OSError:
        return None


def compress(data: bytes) -> bytes:
    return pa.compress(data, codec="snappy", asbytes=True)


class Stream:
    def __init__(self):
        self.elements = bytearray()
        self.expected = bytearray()

    def literal(self, data: bytes, length_bytes: Optional[int] = None) -> "Stream":
        n = len(data) - 1
        assert n >= 0
        if length_bytes is None:
            length_bytes = 0 if n < 60 else (n.bit_length() + 7) // 8
        if length_bytes == 0:
            assert n < 60
            self.elements.append(n << 2)
        else:
            assert 1 <= length_bytes <= 4 and n < 1 << (8 * length_bytes)
            self.elements.append((59 + length_bytes) << 2)
            self.elements += n.to_bytes(length_bytes, "little")
        self.elements += data
        self.expected += data
        return self

    def copy(self, offset: int, length: int, kind: Optional[int] = None) -> "Stream":
        if kind is None:
            kind = 1 if 4 <= length <= 11 and offset < 2048 else (2 if offset < 65536 else 4)
        if kind == 1:
            assert 4 <= length <= 11 and 0 <= offset < 2048
            self.elements += bytes([1 | ((length - 4) << 2) | ((offset >> 8) << 5), offset & 0xFF])
        elif kind == 2:
            assert 1 <= length <= 64 and 0 <= offset < 65536
            self.elements += bytes([2 | ((length - 1) << 2)]) + struct.pack("<H", offset)
        else:
            assert kind == 4 and 1 <= length <= 64 and 0 <= offset < 1 << 32
            self.elements += bytes([3 | ((length - 1) << 2)]) + struct.pack("<I", offset)
        assert 0 < offset <= len(self.expected), "a malformed copy goes in through raw()"
        for _ in range(length):
            self.expected.append(self.expected[-offset])
        return self

    def raw(self, b: bytes) -> "Stream":
        """Bytes appended to the elements as they are (for malformed streams)."""
        self.elements += b
        return self

    def bytes(self, declared: Optional[int] = None) -> bytes:
        return varint(len(self.expected) if declared is None else declared) + bytes(self.elements)


TEXT = bytes((i * 131 + (i >> 7) * 17 + 5) & 255 for i in range(200_000))


def _literal_cases() -> Dict[str, Stream]:
    out = {"inline_1_to_60": Stream()}
    for n in range(1, 61):
        out["inline_1_to_60"].literal(TEXT[n * 61:n * 62], 0)
    for n in (1, 60, 61, 256, 257, 65536, 65537):
        for k in (1, 2, 3, 4):
            if n - 1 < 1 << (8 * k):
                out[f"literal_{n}_in_{k}_length_bytes"] = Stream().literal(TEXT[7:7 + n], k)
    return out


def _copy_cases() -> Dict[str, Stream]:
    out = {}
    s = Stream().literal(TEXT[:2048])
    for o in (1, 2, 7, 8, 255, 256, 1023, 2047):
        for m in range(4, 12):
            s.copy(o, m, 1)
    out["copy1_lengths_4_to_11"] = s
    s = Stream().literal(TEXT[:65535], 2)
    for o in (1, 31, 32, 33, 2048, 65535):
        for m in range(1, 65):
            s.copy(o, m, 2)
    out["copy2_lengths_1_to_64"] = s
    s = Stream().literal(TEXT[:100_000], 3)                 # a page over 64 KiB: copy-4 offsets at and past 65536
    for o in (1, 65535, 65536, 65537, 100_000):
        for m in range(1, 65):
            s.copy(o, m, 4)
    out["copy4_offsets_past_64k"] = s
    for kind in (2, 4):                                      # overlapping copies: offsets 1..33 x lengths 1..64
        s = Stream().literal(TEXT[:40])
        for o in range(1, 34):
            for m in range(1, 65):
                s.copy(o, m, kind)
                s.literal(TEXT[o * 64 + m:o * 64 + m + 3])
        out[f"overlap_copy{kind}_offsets_1_to_33"] = s
    s = Stream().literal(TEXT[:40])
    for o in range(1, 34):
        for m in range(4, 12):
            s.copy(o, m, 1)
    out["overlap_copy1_offsets_1_to_33"] = s
    return out


def _random_stream(seed: int, size: int) -> Stream:
    rng = random.Random(seed)
    s = Stream().literal(TEXT[:64])
    while len(s.expected) < size:
        k = rng.randrange(6)
        if k == 0:
            n = rng.choice([1, 5, 60, 61, 300, 5000])
            a = rng.randrange(len(TEXT) - n)
            s.literal(TEXT[a:a + n], rng.choice([None, 4]) if n <= 60 else None)
        else:
            o = rng.randrange(1, min(len(s.expected), 70_000 if k == 4 else 3000) + 1)
            kind = 4 if k == 4 else (1 if k == 1 and o < 2048 else 2)
            m = rng.randrange(4, 12) if kind == 1 else rng.randrange(1, 65)
            s.copy(o, m, kind)
    return s


def streams() -> Dict[str, Stream]:
    """name -> a well-formed stream of hand-picked elements."""
    out = {}
    out.update(_literal_cases())
    out.update(_copy_cases())
    out["mixed_small"] = _random_stream(1, 3000)
    out["mixed_300k"] = _random_stream(2, 300_000)
    out["empty"] = Stream()
    return out


def _copy36(kind: int, offset: int) -> bytes:
    """56 bytes: a 20-byte literal, then a 36-byte copy-2 or copy-4 element with the given offset."""
    op = struct.pack("<H", offset) if kind == 2 else struct.pack("<I", offset)
    return varint(56) + bytes(Stream().literal(TEXT[:20]).elements) + bytes([(2 if kind == 2 else 3) | (35 << 2)]) + op


def _two_literals(length_bytes: bytes) -> bytes:
    """16 bytes: an 8-byte literal, then a literal whose 4 length bytes (length - 1) are given, then 8 bytes."""
    return varint(16) + bytes(Stream().literal(TEXT[:8]).elements) + b"\xfc" + length_bytes + TEXT[:8]


def refusals() -> Dict[str, tuple]:
    """name -> (stream bytes, output size): one malformed stream per refusal rule; libsnappy refuses each.  Every
    size is a multiple of 8, so each stream can stand for the values of an INT64 page.  Where the fault is one field,
    the stream with only that field corrected fills the size exactly (refusal_controls), so the rule under test is the
    only reason to refuse it."""
    good = Stream().literal(TEXT[:20]).copy(4, 30, 2).literal(TEXT[100:106])
    n = len(good.expected)
    body = bytes(good.elements)
    lit20 = bytes(Stream().literal(TEXT[:20]).elements)
    lit8 = bytes(Stream().literal(TEXT[:8]).elements)
    return {
        "preamble_above_size": (good.bytes(n + 1), n),
        "preamble_below_size": (good.bytes(n - 1), n),
        "offset_0": (_copy36(2, 0), 56),
        "offset_past_output": (_copy36(2, 21), 56),
        "copy4_offset_0": (_copy36(4, 0), 56),
        "copy4_offset_past_output": (_copy36(4, 1 << 31), 56),
        "copy_past_output": (varint(40) + body[:-7], 40),                # 20 literals + a 30-byte copy into 40 bytes
        "literal_past_input": (varint(104) + b"\xf0\x67" + TEXT[:50], 104),
        "literal_past_output": (varint(8) + lit20, 8),
        "int_max_literal": (_two_literals(b"\xfe\xff\xff\x7f"), 16),
        "wrapped_length_literal": (_two_literals(b"\xff\xff\xff\xff"), 16),
        "no_elements": (varint(n), n),
        "empty_input": (b"", 8),
        "truncated_length_bytes": (varint(304) + b"\xf4\x2f", 304),
        "truncated_copy1_operand": (varint(32) + lit8 + b"\x01", 32),
        "truncated_copy2_operand": (varint(32) + lit8 + b"\x3a\x04", 32),
        "truncated_copy4_operand": (varint(32) + lit8 + b"\x3b\x04\x00\x00", 32),
        "preamble_of_6_bytes": (bytes([0x80 | n, 0x80, 0x80, 0x80, 0x80, 0x00]) + body, n),
        "preamble_above_32_bits": (bytes([0x80 | n, 0x80, 0x80, 0x80, 0x10]) + body, n),
        "trailing_elements": (good.bytes() + b"\x00x", n),
    }


def refusal_controls() -> Dict[str, tuple]:
    """name -> (stream bytes, expected output): the refusals whose fault is one field, with that field corrected."""
    good = Stream().literal(TEXT[:20]).copy(4, 30, 2).literal(TEXT[100:106])
    n = len(good.expected)
    copy2 = (_copy36(2, 4), bytes(Stream().literal(TEXT[:20]).copy(4, 36, 2).expected))
    copy4 = (_copy36(4, 4), copy2[1])
    lits = (_two_literals(struct.pack("<I", 7)), TEXT[:8] * 2)
    return {
        "offset_0": copy2, "offset_past_output": copy2, "copy4_offset_0": copy4, "copy4_offset_past_output": copy4,
        "int_max_literal": lits, "wrapped_length_literal": lits,
        "preamble_above_32_bits": (bytes([0x80 | n, 0x80, 0x80, 0x80, 0x00]) + bytes(good.elements),
                                   bytes(good.expected)),
    }


def non_canonical_preamble() -> tuple:
    """A 5-byte preamble for a small size (libsnappy takes it): (stream bytes, expected output)."""
    good = Stream().literal(TEXT[:20]).copy(4, 30, 2).literal(TEXT[100:106])
    n = len(good.expected)
    return bytes([0x80 | n, 0x80, 0x80, 0x80, 0x00]) + bytes(good.elements), bytes(good.expected)
