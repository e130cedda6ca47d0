"""ORC files built stream by stream on the host, for tests that need byte layouts no writer produces on request.

Written from the public ORC specification (v1: file tail, stripes, column encodings, RLE v1 / v2, byte RLE, boolean
streams, decimals, compression chunks) and the protobuf wire format; independent of the repository's ORC reader and
writer (orc_meta.cc, orc_encode_device.cuh), so it can judge the decoder.  The pieces:

  Pb                   protobuf writer: varint, length-delimited, packed repeated fields, nested messages
  short_repeat /       RLE v2 runs, each with explicit header fields (widths, lengths, base bytes, patch and gap widths,
  direct /             patch positions) whose ranges the encoder checks, so a case names the exact run it wants
  patched_base / delta
  rle1_run /           RLE v1 runs and literal groups; byte RLE; boolean bit streams; zigzag varints; DECIMAL values
  rle1_literals / ...
  frame                compression chunks of a stream: original or compressed, cut at given offsets, under ZLIB (raw
                       DEFLATE, fixed-Huffman or stored blocks), ZSTD (one or more frames per chunk) or LZ4 (raw blocks)
  kv_orc_file          a flat KeyValue file [_KEY_pk, _SEQUENCE_NUMBER, _VALUE_KIND, pk, v] whose stripes carry the value
                       column's streams as the case dictates (plus a ROW_INDEX stream readers skip)

Expected values are plain Python values (None = NULL); they are the reference the decoder is compared with.  Floats
are IEEE bit patterns (ints), strings and binaries bytes, DECIMAL values unscaled ints at the column's scale.
"""
import io
import zlib
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
import pyarrow as pa

# orc_proto enums
NONE, ZLIB, SNAPPY, LZO, LZ4, ZSTD = range(6)
K_BOOLEAN, K_BYTE, K_SHORT, K_INT, K_LONG, K_FLOAT, K_DOUBLE, K_STRING, K_BINARY, K_TIMESTAMP = range(10)
K_STRUCT, K_DECIMAL, K_DATE = 12, 14, 15
PRESENT, DATA, LENGTH, DICTIONARY_DATA, DICTIONARY_COUNT, SECONDARY, ROW_INDEX = range(7)
DIRECT, DICTIONARY, DIRECT_V2, DICTIONARY_V2 = range(4)

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def uvarint(v: int) -> bytes:
    assert v >= 0
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def zigzag(v: int) -> int:
    """Zigzag of any Python int (ORC's signed varints are unbounded for DECIMAL)."""
    return 2 * v if v >= 0 else -2 * v - 1


def unzigzag(u: int) -> int:
    return u >> 1 if not u & 1 else -((u + 1) >> 1)


def svarint(v: int) -> bytes:
    return uvarint(zigzag(v))


class Pb:
    """Protobuf wire format: key = field << 3 | wire type; 0 = varint, 2 = length-delimited."""

    def __init__(self):
        self.b = bytearray()

    def key(self, f: int, wire: int):
        self.b += uvarint(f << 3 | wire)

    def u(self, f: int, v: int):
        self.key(f, 0)
        self.b += uvarint(v)

    def bytes(self, f: int, v: bytes):
        self.key(f, 2)
        self.b += uvarint(len(v)) + bytes(v)

    def msg(self, f: int, m: "Pb"):
        self.bytes(f, m.b)

    def packed(self, f: int, vals: Sequence[int]):
        self.bytes(f, b"".join(uvarint(v) for v in vals))


# ------------------------------------------------------------------ RLE v2

FIXED_WIDTHS = list(range(1, 25)) + [26, 28, 30, 32, 40, 48, 56, 64]     # the 5-bit width codes 0..31


def width_code(w: int) -> int:
    assert w in FIXED_WIDTHS, f"{w} bits is not an encodable width"
    return FIXED_WIDTHS.index(w)


def closest_fixed_bits(n: int) -> int:
    return 1 if n == 0 else next(w for w in FIXED_WIDTHS if w >= n)


def pack_be(values: Sequence[int], width: int) -> bytes:
    """Big-endian bit packing, most significant bit first, the last byte padded with zeros."""
    if width == 0 or not values:
        return b""
    acc = 0
    for v in values:
        assert 0 <= v < (1 << width), (v, width)
        acc = (acc << width) | v
    bits = width * len(values)
    pad = (-bits) % 8
    return (acc << pad).to_bytes((bits + pad) // 8, "big")


def _len_bytes(tag: int, code: int, n: int) -> bytes:
    assert 1 <= n <= 512 and 0 <= code <= 31
    return bytes([tag << 6 | code << 1 | (n - 1) >> 8, (n - 1) & 0xFF])


def short_repeat(value: int, width: int, count: int, signed: bool = True):
    """SHORT_REPEAT: `count` (3..10) copies of one value stored in `width` (1..8) big-endian bytes."""
    assert 1 <= width <= 8 and 3 <= count <= 10
    u = zigzag(value) if signed else value
    assert 0 <= u < 1 << (8 * width), (value, width)
    return bytes([(width - 1) << 3 | (count - 3)]) + u.to_bytes(width, "big"), [value] * count


def direct(values: Sequence[int], code: int, signed: bool = True):
    """DIRECT: 1..512 values bit-packed at the width of `code` (0..31)."""
    us = [zigzag(v) if signed else v for v in values]
    return _len_bytes(1, code, len(values)) + pack_be(us, FIXED_WIDTHS[code]), list(values)


def patched_base_raw(n: int, width: int, base_bytes: int, base: int, data: Sequence[int], patch_width: int,
                     gap_width: int, entries: Sequence[int]) -> bytes:
    """PATCHED_BASE header and body from raw fields: no check beyond the header's own bit fields (malformed cases use
    this directly)."""
    assert 1 <= base_bytes <= 8 and 1 <= gap_width <= 8 and len(entries) <= 31
    cfb = closest_fixed_bits(min(patch_width + gap_width, 64))
    mag = abs(base) | ((1 << (8 * base_bytes - 1)) if base < 0 else 0)
    return (_len_bytes(2, width_code(width), n) + bytes([(base_bytes - 1) << 5 | width_code(patch_width),
                                                          (gap_width - 1) << 5 | len(entries)])
            + mag.to_bytes(base_bytes, "big") + pack_be(list(data), width)
            + pack_be(list(entries), cfb))


def patched_base(values: Sequence[int], base_bytes: int, width: int, patch_width: int, gap_width: int,
                 patches: Optional[Sequence[int]] = None, base: Optional[int] = None):
    """PATCHED_BASE: values - base packed at `width` bits; the bits above `width` of the values at `patches` (default:
    those that need them; an explicit list may add positions whose patch is 0) go to the patch list as
    (gap << patch_width | patch) entries of closest_fixed_bits(patch_width + gap_width) bits.  A gap wider than
    gap_width bits becomes filler entries (the largest gap, patch 0) first.  base: default the minimum, stored in
    `base_bytes` bytes, sign and magnitude."""
    n = len(values)
    base = min(values) if base is None else base
    assert 1 <= n <= 512 and 1 <= base_bytes <= 8 and 1 <= gap_width <= 8
    assert width in FIXED_WIDTHS and patch_width in FIXED_WIDTHS and patch_width + gap_width <= 64
    assert abs(base) < 1 << (8 * base_bytes - 1), "the base does not fit its bytes"
    rel = [v - base for v in values]
    assert min(rel) >= 0
    need = [i for i, r in enumerate(rel) if r >> width]
    patches = need if patches is None else sorted(patches)
    assert set(need) <= set(patches) and all(0 <= i < n for i in patches)
    max_gap = (1 << gap_width) - 1
    entries, prev = [], 0
    for i in patches:
        gap = i - prev
        while gap > max_gap:
            entries.append(max_gap << patch_width)
            gap -= max_gap
        p = rel[i] >> width
        assert p < 1 << patch_width, "a patch does not fit the patch width"
        entries.append(gap << patch_width | p)
        prev = i
    assert 1 <= len(entries) <= 31, "the patch list holds 1 to 31 entries"
    mask = (1 << width) - 1
    return patched_base_raw(n, width, base_bytes, base, [r & mask for r in rel], patch_width, gap_width, entries), list(values)


def delta(base: int, delta_base: int, deltas: Optional[Sequence[int]], code: int, signed: bool = True):
    """DELTA: the first value, the delta base (signed; its sign is the direction of every later delta), then the
    magnitudes of deltas 2.. bit-packed at the width of `code` (1..31).  code 0 = fixed delta: no packed deltas, every
    magnitude must equal |delta_base|.  deltas None = a run of one value."""
    n = 1 if deltas is None else 2 + len(deltas)
    deltas = list(deltas or [])
    if code == 0:
        assert all(d == abs(delta_base) for d in deltas)
    else:
        assert all(0 <= d < 1 << FIXED_WIDTHS[code] for d in deltas)
    vals = [base] + ([base + delta_base] if n > 1 else [])
    for d in deltas:
        vals.append(vals[-1] + (d if delta_base >= 0 else -d))
    assert all(INT64_MIN <= v <= INT64_MAX for v in vals)
    head = svarint(base) if signed else uvarint(base)
    body = pack_be(deltas, FIXED_WIDTHS[code]) if code and n > 2 else b""
    return _len_bytes(3, code, n) + head + svarint(delta_base) + body, vals


# ------------------------------------------------------------------ RLE v1, byte RLE, booleans, decimals

def rle1_run(base: int, step: int, count: int, signed: bool = True):
    """RLE v1 run: header count - 3 (count 3..130), a signed delta byte (-128..127), the base as a varint."""
    assert 3 <= count <= 130 and -128 <= step <= 127
    vals = [base + j * step for j in range(count)]
    assert all(INT64_MIN <= v <= INT64_MAX for v in vals)
    return bytes([count - 3, step & 0xFF]) + (svarint(base) if signed else uvarint(base)), vals


def rle1_literals(values: Sequence[int], signed: bool = True):
    """RLE v1 literal group: header 256 - n (n 1..128), then n varints."""
    assert 1 <= len(values) <= 128
    return bytes([256 - len(values)]) + b"".join(svarint(v) if signed else uvarint(v) for v in values), list(values)


def concat(*runs):
    """(bytes, values) runs -> one stream and its values."""
    return b"".join(r[0] for r in runs), [v for r in runs for v in r[1]]


def byte_rle(plan) -> bytes:
    """Byte RLE from an explicit plan: ("run", count 3..130, value) and ("lit", values of 1..128 bytes)."""
    out = bytearray()
    for item in plan:
        if item[0] == "run":
            _, n, v = item
            assert 3 <= n <= 130
            out += bytes([n - 3, v & 0xFF])
        else:
            vals = item[1]
            assert 1 <= len(vals) <= 128
            out += bytes([256 - len(vals)]) + bytes(v & 0xFF for v in vals)
    return bytes(out)


def byte_plan(data: Sequence[int]):
    """A greedy plan: equal bytes in runs of 3 to 130, everything else in literal groups of up to 128."""
    plan, lit, i = [], [], 0
    data = list(data)
    while i < len(data):
        j = i
        while j < len(data) and data[j] == data[i] and j - i < 130:
            j += 1
        if j - i >= 3:
            if lit:
                plan += [("lit", lit[k:k + 128]) for k in range(0, len(lit), 128)]
                lit = []
            plan.append(("run", j - i, data[i]))
            i = j
        else:
            lit.append(data[i])
            i += 1
    plan += [("lit", lit[k:k + 128]) for k in range(0, len(lit), 128)]
    return plan


def bool_stream(bits: Sequence[bool]) -> bytes:
    """A boolean stream: bits most significant first, the last byte padded with zeros, then byte RLE."""
    packed = np.packbits(np.asarray([1 if b else 0 for b in bits], np.uint8), bitorder="big").tolist()
    return byte_rle(byte_plan(packed))


def decimal_data(unscaled: Sequence[int]) -> bytes:
    """DECIMAL DATA: the unscaled values as zigzag varints of any length."""
    return b"".join(svarint(v) for v in unscaled)


def rescale(v: int, s: int, scale: int) -> int:
    """A value of scale s at the column's scale: multiplied up, or divided down truncating toward zero."""
    if s <= scale:
        return v * 10 ** (scale - s)
    q = abs(v) // 10 ** (s - scale)
    return q if v >= 0 else -q


# ------------------------------------------------------------------ compression chunks

def compress(codec: int, raw: bytes, mode: str = "default") -> bytes:
    """One chunk's compressed body.  ZLIB: raw DEFLATE ("fixed": fixed-Huffman blocks only, "stored": stored blocks);
    ZSTD: one frame ("frames2": two frames, each over half the bytes); LZ4: one raw block."""
    if codec == ZLIB:
        co = zlib.compressobj(0 if mode == "stored" else 9, zlib.DEFLATED, -15, 9,
                              zlib.Z_FIXED if mode == "fixed" else zlib.Z_DEFAULT_STRATEGY)
        return co.compress(raw) + co.flush()
    if codec == ZSTD:
        if mode == "frames2":
            h = len(raw) // 2
            return pa.compress(raw[:h], codec="zstd", asbytes=True) + pa.compress(raw[h:], codec="zstd", asbytes=True)
        return pa.compress(raw, codec="zstd", asbytes=True)
    if codec == LZ4:
        return pa.compress(raw, codec="lz4_raw", asbytes=True)
    raise ValueError(f"codec {codec}")


def chunk_header(length: int, original: bool) -> bytes:
    assert length < 1 << 23
    return (length << 1 | int(original)).to_bytes(3, "little")


def frame(raw: bytes, codec: int, block: int, plan=None) -> bytes:
    """A stream (or a metadata section) as compression chunks.  plan: [(raw bytes, mode)] cuts the first bytes into
    chunks, mode "original", "compressed", "auto" (compressed unless that is not smaller) or a codec mode of compress();
    the bytes left over are cut every `block` bytes, "auto".  A chunk never inflates to more than `block` bytes."""
    if codec == NONE:
        return raw
    out, pos = bytearray(), 0
    plan = list(plan or [])
    while pos < len(raw):
        n, mode = plan.pop(0) if plan else (min(block, len(raw) - pos), "auto")
        n = min(n, len(raw) - pos)
        assert 0 < n <= block
        part = raw[pos:pos + n]
        if mode == "original":
            out += chunk_header(n, True) + part
        else:
            c = compress(codec, part, mode if mode not in ("auto", "compressed") else "default")
            if mode == "auto" and len(c) >= n:
                out += chunk_header(n, True) + part
            else:
                out += chunk_header(len(c), False) + c
        pos += n
    return bytes(out)


# ------------------------------------------------------------------ files

@dataclass
class VType:
    """The ORC type of the value column and the Paimon type it is read as."""
    read: str                       # Paimon type name
    kind: int
    width: int                      # bytes of the decoded value (0 = var-len)
    precision: int = 0
    scale: int = 0


VTYPES = {
    "BOOLEAN": VType("BOOLEAN", K_BOOLEAN, 1), "TINYINT": VType("TINYINT", K_BYTE, 1),
    "SMALLINT": VType("SMALLINT", K_SHORT, 2), "INT": VType("INT", K_INT, 4), "DATE": VType("DATE", K_DATE, 4),
    "BIGINT": VType("BIGINT", K_LONG, 8), "FLOAT": VType("FLOAT", K_FLOAT, 4), "DOUBLE": VType("DOUBLE", K_DOUBLE, 8),
    "STRING": VType("STRING", K_STRING, 0), "BINARY": VType("BINARY", K_BINARY, 0),
    "DECIMAL(10,5)": VType("DECIMAL(10,5)", K_DECIMAL, 8, 10, 5),
}


@dataclass
class Stream:
    kind: int
    data: bytes
    plan: object = None             # compression chunk plan (see frame); "asis": the bytes are already chunks


@dataclass
class Stripe:
    """One stripe of the value column: its rows, expected values (None = NULL), encoding and streams."""
    values: list
    streams: List[Stream]
    encoding: int = DIRECT_V2
    dict_size: int = 0
    row_index: bool = True


@dataclass
class OrcFile:
    data: bytes
    expected: list
    n_tasks: int                    # (stripe, column) tasks of the five columns
    n_streams: int                  # non-empty PRESENT / DATA / LENGTH / DICTIONARY_DATA / SECONDARY streams


def present(values) -> List[Stream]:
    """The PRESENT stream of a stripe's values, or nothing when every value is there."""
    if all(v is not None for v in values):
        return []
    return [Stream(PRESENT, bool_stream([v is not None for v in values]))]


def _key_stream(first: int, n: int) -> bytes:
    """first, first + 1, ... as fixed-delta DELTA runs of up to 512 values."""
    out = bytearray()
    for s in range(0, n, 512):
        m = min(512, n - s)
        out += delta(first + s, 1, [1] * (m - 2), 0)[0] if m >= 2 else direct([first + s], 31)[0]
    return bytes(out)


def _zero_bytes(n: int) -> bytes:
    return byte_rle([("run", min(130, n - s), 0) if n - s >= 3 else ("lit", [0] * (n - s)) for s in range(0, n, 130)])


def _stream_msg(kind, column, length) -> Pb:
    m = Pb()
    m.u(1, kind)
    m.u(2, column)
    m.u(3, length)
    return m


def kv_orc_file(vt: VType, stripes: Sequence[Stripe], codec: int = NONE, block: int = 262144, key0: int = 0,
                footer_dict_size: Optional[dict] = None) -> OrcFile:
    """A flat KeyValue ORC file [_KEY_pk LONG, _SEQUENCE_NUMBER LONG, _VALUE_KIND BYTE, pk LONG, v] whose stripes hold
    the given value-column stripes.  pk = key0 + row, _SEQUENCE_NUMBER = row, _VALUE_KIND = 0.  Every stripe's index
    section holds a ROW_INDEX stream for v (when the stripe asks for one).  footer_dict_size: {stripe: n} overrides the
    dictionarySize a stripe footer claims."""
    names = [b"_KEY_pk", b"_SEQUENCE_NUMBER", b"_VALUE_KIND", b"pk", b"v"]
    out = bytearray(b"ORC")
    infos, row, n_streams = [], 0, 0
    for si, st in enumerate(stripes):
        n = len(st.values)
        assert n > 0
        keys = _key_stream(key0 + row, n)
        index, data = [], [(1, DATA, keys, None), (2, DATA, _key_stream(row, n), None), (3, DATA, _zero_bytes(n), None),
                           (4, DATA, keys, None)]
        if st.row_index:
            ri = Pb()                                   # RowIndex { RowIndexEntry { positions } }
            e = Pb()
            e.packed(1, [0, 0, 0])
            ri.msg(1, e)
            index.append((5, ROW_INDEX, bytes(ri.b), None))
        data += [(5, s.kind, s.data, s.plan) for s in st.streams]
        offset = len(out)
        footer = Pb()
        lengths = []
        for part in (index, data):
            start = len(out)
            for col, kind, raw, plan in part:
                stored = raw if plan == "asis" else frame(raw, codec, block, plan)
                out += stored
                footer.msg(1, _stream_msg(kind, col, len(stored)))
                if kind != ROW_INDEX and len(stored):
                    n_streams += 1
            lengths.append(len(out) - start)
        for col in range(6):
            e = Pb()
            if col == 5:
                e.u(1, st.encoding)
                ds = (footer_dict_size or {}).get(si, st.dict_size)
                if st.encoding in (DICTIONARY, DICTIONARY_V2) or ds:
                    e.u(2, ds)
            else:
                e.u(1, DIRECT if col in (0, 3) else DIRECT_V2)
            footer.msg(2, e)
        fbytes = frame(bytes(footer.b), codec, block)
        out += fbytes
        infos.append((offset, lengths[0], lengths[1], len(fbytes), n))
        row += n
    content = len(out)
    ft = Pb()
    ft.u(1, 3)                                           # headerLength
    ft.u(2, content)                                     # contentLength
    for off, il, dl, fl, n in infos:
        s = Pb()
        s.u(1, off)
        s.u(2, il)
        s.u(3, dl)
        s.u(4, fl)
        s.u(5, n)
        ft.msg(3, s)
    root = Pb()
    root.u(1, K_STRUCT)
    root.packed(2, [1, 2, 3, 4, 5])
    for nm in names:
        root.bytes(3, nm)
    ft.msg(4, root)
    for kind in (K_LONG, K_LONG, K_BYTE, K_LONG, vt.kind):
        t = Pb()
        t.u(1, kind)
        if kind == K_DECIMAL:
            t.u(5, vt.precision)
            t.u(6, vt.scale)
        ft.msg(4, t)
    ft.u(6, row)                                         # numberOfRows
    ft.u(8, 10000)                                       # rowIndexStride
    fb = frame(bytes(ft.b), codec, block)
    out += fb
    ps = Pb()                                            # PostScript
    ps.u(1, len(fb))
    ps.u(2, codec)
    if codec != NONE:
        ps.u(3, block)
    ps.packed(4, [0, 12])
    ps.u(5, 0)                                           # metadataLength: no stripe statistics
    ps.u(6, 6)                                           # writerVersion
    ps.bytes(8000, b"ORC")
    assert len(ps.b) < 256
    out += ps.b + bytes([len(ps.b)])
    expected = [v for st in stripes for v in st.values]
    return OrcFile(bytes(out), expected, 5 * len(stripes), n_streams)


# ------------------------------------------------------------------ cases
#
# A case is the files of one sorted run and the values "v" must decode to.

@dataclass
class Case:
    name: str
    files: List[OrcFile]
    vtype: str                      # key of VTYPES
    pyarrow: bool = True            # pyarrow reads the files (False: a layout the spec allows and pyarrow refuses)
    codec: int = NONE
    arrow_view: object = None       # expected value -> what pyarrow's reading holds, where the two differ by design

    @property
    def expected(self):
        return [v for f in self.files for v in f.expected]

    @property
    def n_tasks(self):
        return sum(f.n_tasks for f in self.files)

    @property
    def n_streams(self):
        return sum(f.n_streams for f in self.files)


def with_nulls(values: Sequence, pattern) -> list:
    """values spread over rows: row r is NULL where pattern(r) is true, until every value is placed."""
    out, it, r = [], iter(values), 0
    left = len(values)
    while left:
        if pattern(r):
            out.append(None)
        else:
            out.append(next(it))
            left -= 1
        r += 1
    return out


def int_stripes(vt: VType, runs, per_stripe: int, encoding=DIRECT_V2, null_every: int = 0, plans=None) -> List[Stripe]:
    """Integer runs [(bytes, values)] over stripes of `per_stripe` runs; with null_every, every odd stripe has a NULL
    at each row r with r % null_every == 1."""
    stripes = []
    for k, s in enumerate(range(0, len(runs), per_stripe)):
        data, vals = concat(*runs[s:s + per_stripe])
        if null_every and k % 2:
            vals = with_nulls(vals, lambda r: r % null_every == 1)
        stripes.append(Stripe(vals, present(vals) + [Stream(DATA, data, plans[k] if plans else None)], encoding))
    return stripes


def short_repeat_case() -> Case:
    """SHORT_REPEAT at every value width (1..8 bytes, the value needing exactly that many, plus 0 and INT64_MIN at 8)
    and every count (3..10)."""
    runs = []
    for w in range(1, 9):
        for c in range(3, 11):
            u = (1 << (8 * w - 1)) | (c * 37 + w) if w > 1 else 0x80 | c
            runs.append(short_repeat(unzigzag(u), w, c))
    runs += [short_repeat(0, 8, 3), short_repeat(INT64_MIN, 8, 10), short_repeat(INT64_MAX, 8, 4)]
    return Case("rle2_short_repeat", [kv_orc_file(VTYPES["BIGINT"], int_stripes(VTYPES["BIGINT"], runs, 20, null_every=5))], "BIGINT")


def _direct_vals(w: int, n: int, rng, signed=True):
    """n values whose zigzag (or unsigned value) needs `w` bits, the largest of the width among them."""
    top = (1 << w) - 1
    us = [int(x) for x in rng.integers(0, top, n, endpoint=True, dtype=np.uint64)]
    us[n // 2] = top
    return [unzigzag(u) for u in us] if signed else us


def direct_case(vtype: str = "BIGINT") -> Case:
    """DIRECT at each of the 32 width codes (26 to 64 bits included; INT / SMALLINT / DATE stop at their type's width)
    with lengths 1, 37, 512 and 255 in turn."""
    vt = VTYPES[vtype]
    bits = 8 * vt.width
    rng = np.random.default_rng(bits)
    runs = []
    for code, w in enumerate(FIXED_WIDTHS):
        n = [1, 37, 512, 255][code % 4]
        vw = min(w, bits)                               # values of a narrower type at a wider width: legal
        runs.append(direct(_direct_vals(vw, n, rng), code))
    return Case(f"rle2_direct_{vtype}", [kv_orc_file(vt, int_stripes(vt, runs, 11, null_every=3))], vtype)


def patched_base_case() -> Case:
    """PATCHED_BASE: gap fillers (a patch gap of 300 under 8-bit gaps, 140 under 3-bit gaps), base widths 1 to 8 bytes with
    negative and positive bases, patch + gap widths of 64, 56, 43, 33 and 25 (entries rounded up to 64, 56, 48, 40 and
    26 bits), an explicit patch whose value is 0, and runs of 1, 512 and odd lengths."""
    rng = np.random.default_rng(7)
    runs = []
    # gap fillers: 512 values of 4 bits, patched at 0, 300 (gap 300 = 255 + 45) and 511
    vals = [1000 + int(x) for x in rng.integers(0, 16, 512)]
    for i, p in ((0, 5), (300, 0xABCDE), (511, 1)):
        vals[i] = 1000 + (p << 4 | (vals[i] - 1000))
    vals[100] = 1000                                    # the minimum is the base
    runs.append(patched_base(vals, 2, 4, 20, 8, patches=[0, 300, 511]))
    vals = [-50 + int(x) for x in rng.integers(0, 8, 200)]
    vals[10] = -50
    vals[150] = -50 + (3 << 3 | 5)
    runs.append(patched_base(vals, 1, 3, 2, 3, patches=[10, 150]))       # gap 10, then 140 = 7 * 20 fillers
    # base widths 1..8 bytes, alternating sign; the base at the edge of its bytes
    for bb in range(1, 9):
        base = (1 << (8 * bb - 1)) - 1 if bb % 2 else -((1 << (8 * bb - 1)) - 1)
        base = max(min(base, INT64_MAX - (1 << 40)), -(1 << 62))
        n = [1, 9, 100, 511][bb % 4]
        vals = [base + int(x) for x in rng.integers(0, 1 << 5, n)]
        vals[0] = base
        vals[n - 1] = base + (0x1F << 5 | 3)
        runs.append(patched_base(vals, bb, 5, 5, 8, patches=sorted({0, n - 1}), base=base))
    # patch + gap widths near 64 and closest_fixed_bits rounding of the entries
    for pw, pgw, w, at in ((56, 8, 2, [3, 40, 63]), (48, 8, 6, [0, 63]), (40, 3, 16, [3, 10, 17]),
                           (30, 3, 24, [1, 8]), (24, 1, 32, [0, 1, 2]), (20, 5, 12, [5, 36, 63])):
        n = 64
        base = -12345
        vals = [base + int(x) for x in rng.integers(0, 1 << w, n, dtype=np.uint64)]
        vals[50] = base
        for a in at:
            vals[a] = base + (((1 << pw) - 1 - a) << w | 1)
        runs.append(patched_base(vals, 8, w, pw, pgw, patches=at, base=base))
    # a patch whose value is 0 (the position is listed, its high bits are empty)
    vals = [int(x) for x in rng.integers(0, 1 << 10, 30)]
    vals[0] = 0
    vals[20] = 7 << 10
    runs.append(patched_base(vals, 1, 10, 3, 4, patches=[5, 20], base=0))
    return Case("rle2_patched_base", [kv_orc_file(VTYPES["BIGINT"], int_stripes(VTYPES["BIGINT"], runs, 6, null_every=4))], "BIGINT")


def delta_case() -> Case:
    """DELTA: fixed delta (width 0) up and down, runs of 2 and 512 values, a negative delta base with packed
    deltas, and packed deltas at every width code 1..31."""
    rng = np.random.default_rng(11)
    runs = [delta(5, 3, [3] * 510, 0), delta(-7, -11, [11] * 100, 0), delta(INT64_MAX, 0, [0] * 8, 0),
            delta(-5, 1000, [], 0), delta(77, -1, [], 4)]
    for code in range(1, 32):
        w = FIXED_WIDTHS[code]
        n = [2, 3, 512, 100][code % 4]
        lim = min((1 << w) - 1, (1 << 62) // max(n, 1))
        ds = [int(x) for x in rng.integers(0, lim, n - 2, endpoint=True, dtype=np.uint64)] if n > 2 else []
        if ds:
            ds[0] = lim
        down = code % 2 == 1
        runs.append(delta((1 << 62) if down else -(1 << 62), -5 if down else 5, ds, code))
    return Case("rle2_delta", [kv_orc_file(VTYPES["BIGINT"], int_stripes(VTYPES["BIGINT"], runs, 9, null_every=6))], "BIGINT")


def delta_one_case() -> Case:
    """DELTA runs of one value (a header length of 1, then the first value and a delta base), between other runs.
    The specification allows runs of 1 to 512 values; the ORC C++ reader behind pyarrow refuses a DELTA run of 1
    ("Illegal run length for delta encoding"), so the builder's values are the only oracle here."""
    runs = [delta(42, 9, None, 0), short_repeat(-3, 1, 3), delta(INT64_MIN, 1, None, 7), delta(INT64_MAX, -1, None, 31),
            direct([1, 2, 3], 2)]
    return Case("rle2_delta_length_1", [kv_orc_file(VTYPES["BIGINT"], int_stripes(VTYPES["BIGINT"], runs, 5))],
                "BIGINT", pyarrow=False)


def rle_v1_case() -> Case:
    """RLE v1: runs of 3, 4, 10, 127, 128, 129 and 130 values with deltas -128, -1, 0, 1 and 127; literal groups of
    1, 2, 3, 64, 127 and 128 values; varints of 9 and 10 bytes (zigzag of 2^60, INT64_MIN, INT64_MAX) in literals and
    as run bases."""
    rng = np.random.default_rng(13)
    runs = []
    for i, count in enumerate((3, 4, 10, 127, 128, 129, 130)):
        for step in (-128, -1, 0, 1, 127):
            runs.append(rle1_run(int(rng.integers(-(1 << 40), 1 << 40)), step, count))
        runs.append(rle1_literals([int(x) for x in rng.integers(-(1 << 62), 1 << 62, [1, 2, 3, 64, 127, 128, 5][i])]))
    runs += [rle1_literals([INT64_MIN, INT64_MAX, 1 << 60, -(1 << 60), 0, -1]), rle1_run(INT64_MIN, 0, 5),
             rle1_run(INT64_MAX, -1, 130), rle1_run(INT64_MIN, 127, 3), rle1_run((1 << 60), -128, 100)]
    return Case("rle1", [kv_orc_file(VTYPES["BIGINT"], int_stripes(VTYPES["BIGINT"], runs, 10, DIRECT, null_every=7))], "BIGINT")


def narrow_ints_case(vtype: str) -> Case:
    """SMALLINT / INT / DATE at the type's edges: SHORT_REPEAT (wider than needed), fixed and packed DELTA and
    PATCHED_BASE stripes under RLE v2, and a last stripe under RLE v1 (DIRECT)."""
    vt = VTYPES[vtype]
    bits = 8 * vt.width
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    runs = [short_repeat(lo, (bits + 8) // 8 if bits < 64 else 8, 5), short_repeat(hi, vt.width, 10),
            delta(lo, 1, [1] * 98, 0), delta(hi, -(1 << (bits - 2)), [1 << (bits - 3)] * 2, width_code(closest_fixed_bits(bits - 2))),
            patched_base([lo, lo + 3, lo + 1, hi - 1, lo + 2], 8 if bits > 16 else 3, 2, closest_fixed_bits(bits), 2)]
    st = int_stripes(vt, runs, 3, null_every=4)
    v1 = concat(rle1_run(lo, 127, 4), rle1_literals([lo, hi, 0, -1]), rle1_run(hi, -128, 3))
    st.append(Stripe(v1[1], [Stream(DATA, v1[0])], DIRECT))
    return Case(f"narrow_{vtype}", [kv_orc_file(vt, st)], vtype)


def tinyint_case() -> Case:
    """Byte RLE: runs of 3 to 130 and literal groups of 1 to 128 over stripes of 13, 37, 1001 and 8 rows, NULLs in
    runs that cross the stripe boundaries."""
    stripes, r = [], 0
    for n, plan in ((13, [("run", 3, -128), ("lit", [127]), ("run", 4, 0)]),
                    (37, [("lit", list(range(-5, 20))), ("run", 10, 7)]),
                    (1001, [("run", 130, 1), ("lit", [(i * 37) % 256 - 128 for i in range(128)]), ("run", 129, -1),
                            ("lit", [5, 6]), ("run", 3, 9)]),
                    (8, [("lit", [1, 2, 3])])):
        vals = [((v & 0xFF) ^ 0x80) - 0x80 for item in plan for v in ([item[2]] * item[1] if item[0] == "run" else item[1])]
        it = iter(vals)
        rows = [next(it) if ok else None for ok in _fit_nulls(len(vals), n, r, 50, 40)]
        stripes.append(Stripe(rows, present(rows) + [Stream(DATA, byte_rle(plan))], DIRECT))
        r += n
    return Case("byte_rle", [kv_orc_file(VTYPES["TINYINT"], stripes)], "TINYINT")


def _fit_nulls(vals_n: int, rows: int, start: int, period: int, nulls_at: int):
    """A NULL pattern over `rows` rows with exactly vals_n values: NULL where (start + r) % period >= nulls_at, then
    adjusted at the end."""
    valid = [(start + r) % period < nulls_at for r in range(rows)]
    k = sum(valid)
    i = rows - 1
    while k != vals_n:
        if k < vals_n and not valid[i]:
            valid[i] = True
            k += 1
        elif k > vals_n and valid[i]:
            valid[i] = False
            k -= 1
        i -= 1
    return valid


def boolean_case() -> Case:
    """BOOLEAN over stripes of 1, 7, 9, 13 and 1001 rows: value and PRESENT bit counts that are not multiples of 8, and
    NULL runs (a period of 50 rows, 20 of them NULL) that cross the stripe boundaries."""
    stripes, r = [], 0
    rng = np.random.default_rng(17)
    for n in (1, 7, 9, 13, 1001):
        valid = [(r + q) % 50 < 30 for q in range(n)]
        if n == 1:
            valid = [True]
        bits = [bool(x) for x in rng.integers(0, 2, sum(valid))]
        it = iter(bits)
        rows = [next(it) if ok else None for ok in valid]
        stripes.append(Stripe(rows, present(rows) + ([Stream(DATA, bool_stream(bits))] if bits else []), DIRECT))
        r += n
    return Case("boolean", [kv_orc_file(VTYPES["BOOLEAN"], stripes)], "BOOLEAN")


F32_EDGES = [0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x7FC00001, 0xFFC12345, 0x7F7FFFFF, 0x3F800000, 0]
F64_EDGES = [0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 0x1, 0x7FF8000000000001,
             0xFFF8123456789ABC, 0x7FEFFFFFFFFFFFFF, 0x3FF0000000000000, 0]


def quiet_f32(bits):
    """A FLOAT bit pattern as it comes out of a round trip through double: signalling NaNs quieted."""
    return bits | 0x400000 if bits is not None and (bits & 0x7F800000) == 0x7F800000 and bits & 0x7FFFFF else bits


def float_case(vtype: str) -> Case:
    """FLOAT / DOUBLE: little-endian IEEE values with NaN payloads, signed zeros, infinities and subnormals, NULLs in
    between, over stripes of 3, 64 and 777 rows.  The decoder keeps every bit.  The ORC C++ reader behind pyarrow
    widens FLOAT to double and narrows it back, which quiets signalling NaNs: FLOAT is compared with pyarrow after
    the same quieting."""
    w = VTYPES[vtype].width
    edges = F32_EDGES if w == 4 else F64_EDGES
    rng = np.random.default_rng(w)
    stripes = []
    for k, n in enumerate((3, 64, 777)):
        bits = edges + [int(x) for x in rng.integers(0, (1 << (8 * w)) - 1, n, dtype=np.uint64)]
        rows = with_nulls(bits, lambda r: r % 5 == 4 and k)[:n]
        vals = [v for v in rows if v is not None]
        stripes.append(Stripe(rows, present(rows) + [Stream(DATA, b"".join(v.to_bytes(w, "little") for v in vals))], DIRECT))
    return Case(f"float_{vtype}", [kv_orc_file(VTYPES[vtype], stripes)], vtype,
                arrow_view=quiet_f32 if w == 4 else None)


def decimal_case(v2: bool) -> Case:
    """DECIMAL(10,5) with per-value scales 0..10: scales below the column's are multiplied up (1.50000 stored as 15 at
    scale 1, as orc-core writes a HiveDecimal with its trailing zeros removed), scales above it divided down, truncating
    toward zero, as the ORC C++ reader does.  SECONDARY under RLE v2 (SHORT_REPEAT, DIRECT, DELTA runs) or v1."""
    vt = VTYPES["DECIMAL(10,5)"]
    rng = np.random.default_rng(19 + v2)
    stripes = []
    for k in range(3):
        n = [40, 300, 9][k]
        scales = [int(s) for s in rng.integers(0, 11, n)]
        unscaled = []
        for i, s in enumerate(scales):
            lim = 10 ** (5 + s)                         # |value| < 10^10 at the column's scale
            unscaled.append(int(rng.integers(-lim, lim)))
        if k == 0:
            scales[:6] = [1, 0, 5, 6, 10, 10]
            unscaled[:6] = [15, -99999, -123456789, -7, 99999999999, -99999999999]
        if v2:
            sec = b""
            runs = []
            for s0 in range(0, n, 20):
                part = scales[s0:s0 + 20]
                runs.append(short_repeat(part[0], 1, len(part)) if len(set(part)) == 1 and 3 <= len(part) <= 10
                            else direct(part, width_code(5)))
            sec, got = concat(*runs)
        else:
            sec, got = concat(*[rle1_literals(scales[s0:s0 + 128]) for s0 in range(0, n, 128)])
        assert got == scales
        vals = [rescale(v, s, vt.scale) for v, s in zip(unscaled, scales)]
        rows = [None if i is None else vals[i] for i in with_nulls(list(range(n)), lambda r: r % 6 == 2 and k != 2)]
        streams = present(rows) + [Stream(DATA, decimal_data(unscaled)), Stream(SECONDARY, sec)]
        stripes.append(Stripe(rows, streams, DIRECT_V2 if v2 else DIRECT))
    return Case(f"decimal_scales_{'v2' if v2 else 'v1'}", [kv_orc_file(vt, stripes)], "DECIMAL(10,5)")


def _ulen_stream(lengths, v2: bool, kind: str = "direct"):
    """Unsigned lengths as RLE v2 DIRECT / PATCHED_BASE runs or RLE v1 literals."""
    runs = []
    for s in range(0, len(lengths), 128 if not v2 else 512):
        part = lengths[s:s + (128 if not v2 else 512)]
        if not v2:
            runs.append(rle1_literals(part, signed=False))
        elif kind == "patched" and len(part) >= 2 and max(part) >= 64:
            w = 4
            runs.append(patched_base(part, 1, w, closest_fixed_bits(max(part).bit_length() - w), 8, base=0))
        else:
            runs.append(direct(part, width_code(closest_fixed_bits(max(part).bit_length())), signed=False))
    data, got = concat(*runs)
    assert got == list(lengths)
    return data


def dictionary_case(v2: bool) -> Case:
    """DICTIONARY (v1) / DICTIONARY_V2 strings: a dictionary with an empty entry and a 300-byte one, a dictionary of
    size 1, a dictionary whose only entry is empty, and a stripe whose rows are all NULL that still carries a
    dictionary (its DATA stream empty)."""
    enc = DICTIONARY_V2 if v2 else DICTIONARY
    rng = np.random.default_rng(23 + v2)
    dicts = [[b"", b"alpha", b"\x00\xff\x01", b"x" * 300, b"beta", b"gamma"], [b"only"], [b""], [b"kept"]]
    stripes = []
    for k, entries in enumerate(dicts):
        n = [200, 50, 33, 17][k]
        if k == 3:
            rows = [None] * n
            ids = []
        else:
            ids = [int(x) for x in rng.integers(0, len(entries), n - n // 4)]
            rows = with_nulls(ids, lambda r: r % 4 == 3)
            rows = [None if i is None else entries[i] for i in rows]
        if ids:
            data = concat(*[direct(ids[s:s + 512], 2, signed=False) for s in range(0, len(ids), 512)])[0] if v2 else \
                concat(*[rle1_literals(ids[s:s + 128], signed=False) for s in range(0, len(ids), 128)])[0]
        else:
            data = b""
        streams = present(rows) + [Stream(DATA, data), Stream(LENGTH, _ulen_stream([len(e) for e in entries], v2)),
                                   Stream(DICTIONARY_DATA, b"".join(entries))]
        stripes.append(Stripe(rows, streams, enc, dict_size=len(entries)))
    return Case(f"dictionary_{'v2' if v2 else 'v1'}", [kv_orc_file(VTYPES["STRING"], stripes)], "STRING")


def direct_strings_case(vtype: str, v2: bool) -> Case:
    """DIRECT / DIRECT_V2 strings and binaries with empty values and NULLs; v2 lengths partly PATCHED_BASE (mostly
    short values, a few long ones)."""
    rng = np.random.default_rng(29 + v2)
    stripes = []
    for k, n in enumerate((1, 150, 600)):
        vals = []
        for i in range(n):
            ln = int(rng.integers(0, 12)) if i % 97 != 5 else 700 + i
            body = bytes(int(x) for x in rng.integers(0, 256, ln)) if vtype == "BINARY" else (b"s%d-" % i * 200)[:ln]
            vals.append(body)
        rows = with_nulls(vals, lambda r: r % 7 == 3 and k)[:n]
        vals = [v for v in rows if v is not None]
        streams = present(rows) + [Stream(DATA, b"".join(vals)),
                                   Stream(LENGTH, _ulen_stream([len(v) for v in vals], v2, "patched" if k == 2 else "direct"))]
        stripes.append(Stripe(rows, streams, DIRECT_V2 if v2 else DIRECT))
    return Case(f"direct_{vtype}_{'v2' if v2 else 'v1'}", [kv_orc_file(VTYPES[vtype], stripes)], vtype)


def compression_case(codec: int) -> Case:
    """Compression chunks of one stream: an original chunk of 1 byte (it splits the 2-byte DIRECT header), a
    compressed chunk cut in the middle of a packed value, a compressed chunk that inflates to exactly the block size,
    original and compressed chunks alternating; ZLIB adds fixed-Huffman and stored DEFLATE blocks, ZSTD a chunk of two
    frames.  A second stripe carries RLE v1 varints cut inside a varint, and strings whose PRESENT, LENGTH and DATA
    streams are framed the same way (STRING file: the LENGTH cut inside a run header)."""
    block = 4096
    mode2 = {ZLIB: "fixed", ZSTD: "frames2", LZ4: "compressed"}[codec]
    mode3 = {ZLIB: "stored", ZSTD: "compressed", LZ4: "compressed"}[codec]
    plan = [(1, "original"), (1000, "compressed"), (block, "compressed"), (77, "original"), (600, mode2),
            (block, mode3), (3, "compressed"), (block - 1, "original")]
    # compressible 64-bit values: a repeating pattern so chunks shrink
    pat = [unzigzag(0x0123456789ABCDEF ^ (i % 5)) for i in range(512)]
    runs = [direct(pat, 31) for _ in range(5)]
    data, vals = concat(*runs)
    st = [Stripe(vals, [Stream(DATA, data, plan)])]
    v1 = concat(*[rle1_literals([INT64_MIN + i, (1 << 60) + i, -i]) for i in range(40)])
    # a 10-byte varint starts at byte 1 of every group: cut at 5 lands inside it
    rows = with_nulls(v1[1], lambda r: r % 3 == 0)
    st.append(Stripe(rows, [Stream(PRESENT, bool_stream([v is not None for v in rows]), [(1, "original"), (2, "compressed")]),
                            Stream(DATA, v1[0], [(5, "compressed"), (12, "original"), (30, "compressed")])], DIRECT))
    f1 = kv_orc_file(VTYPES["BIGINT"], st, codec=codec, block=block)
    # strings under the same codec
    strs = [[b"", b"abc" * (i % 40), bytes([i & 255]) * (i % 7)][i % 3] for i in range(300)]
    rows = with_nulls(strs, lambda r: r % 9 == 8)
    lens = _ulen_stream([len(s) for s in strs], True)
    f2 = kv_orc_file(VTYPES["STRING"], [Stripe(rows, [Stream(PRESENT, bool_stream([v is not None for v in rows]), [(3, "compressed")]),
                                                      Stream(DATA, b"".join(strs), [(100, "original"), (2000, "compressed")]),
                                                      Stream(LENGTH, lens, [(1, "original"), (1, "compressed")])])],
                     codec=codec, block=block)
    name = {ZLIB: "zlib", ZSTD: "zstd", LZ4: "lz4"}[codec]
    return [Case(f"chunks_{name}", [f1], "BIGINT", codec=codec), Case(f"chunks_{name}_strings", [f2], "STRING", codec=codec)]


JOIN_STRIPES = [1, 7, 31, 32, 33, 4095]


def validity_join_case() -> Case:
    """One run of four files whose stripes hold 1, 7, 31, 32, 33 and 4,095 rows (rotated per file): stripe and file
    starts fall inside validity words, so neighbouring stripes and files OR their bits into shared words.  Each file
    has a stripe without NULLs (no PRESENT stream) and one whose rows are all NULL (no DATA stream)."""
    rng = np.random.default_rng(37)
    files, key0 = [], 0
    for fi in range(4):
        sizes = JOIN_STRIPES[fi:] + JOIN_STRIPES[:fi]
        stripes = []
        for k, n in enumerate(sizes):
            if k == 1:
                valid = [True] * n
            elif k == 2:
                valid = [False] * n
            else:
                valid = [(r * 7 + k + fi) % 3 != 0 for r in range(n)]
            vals = [int(x) for x in rng.integers(-(1 << 40), 1 << 40, sum(valid))]
            it = iter(vals)
            rows = [next(it) if ok else None for ok in valid]
            data = concat(*[direct(vals[s:s + 512], width_code(48)) for s in range(0, len(vals), 512)])[0] if vals else b""
            stripes.append(Stripe(rows, present(rows) + [Stream(DATA, data)]))
        files.append(kv_orc_file(VTYPES["BIGINT"], stripes, key0=key0))
        key0 += len(files[-1].expected)
    return Case("validity_join", files, "BIGINT")


MANY_STRIPES, MANY_PER_FILE = 300, 25
MANY_CODECS = [ZLIB, ZSTD, LZ4, NONE]


def many_streams_dictionary(k: int) -> List[bytes]:
    """The dictionary of stripe k: 1,500 random letters (under ZSTD: Huffman-coded literals, 4 streams), a period-5
    pattern of 500 bytes (matches longer than 32 bytes whose offset, 5, is shorter than the match; under ZLIB a match
    distance shorter than its length), an empty entry and one byte."""
    rng = np.random.default_rng(1000 + k)
    return [bytes(int(x) for x in rng.integers(97, 123, 1500)), b"abcde" * 100, b"", b"q"]


def many_streams_case() -> Case:
    """300 stripes of 20 rows in 12 files, ZLIB, ZSTD, LZ4 and uncompressed files in turn within one run; each stripe
    has 8 streams (4 key columns; PRESENT, DATA, LENGTH and DICTIONARY_DATA of a DICTIONARY_V2 string), 2,400 in all:
    more than one per warp of the device's stream decode, so warps decode several streams of different codecs."""
    files, key0 = [], 0
    for f0 in range(0, MANY_STRIPES, MANY_PER_FILE):
        stripes = []
        for k in range(f0, f0 + MANY_PER_FILE):
            entries = many_streams_dictionary(k)
            valid = [(r + k) % 5 != 0 for r in range(20)]
            ids = [(r * 3 + k) % 4 for r in range(sum(valid))]
            it = iter(ids)
            rows = [entries[next(it)] if ok else None for ok in valid]
            streams = present(rows) + [Stream(DATA, direct(ids, width_code(2), signed=False)[0]),
                                       Stream(LENGTH, direct([len(e) for e in entries], width_code(12), signed=False)[0]),
                                       Stream(DICTIONARY_DATA, b"".join(entries))]
            stripes.append(Stripe(rows, streams, DICTIONARY_V2, dict_size=len(entries)))
        files.append(kv_orc_file(VTYPES["STRING"], stripes, codec=MANY_CODECS[(f0 // MANY_PER_FILE) % 4], key0=key0))
        key0 += len(files[-1].expected)
    return Case("many_streams", files, "STRING", codec=LZ4)


def zstd_literals_streams(frame_bytes: bytes) -> int:
    """The number of Huffman streams (1 or 4) of the first block's literals of a zstd frame, 0 when they are not
    Huffman-coded (RFC 8878 sections 3.1.1.1, 3.1.1.2 and 3.1.1.3.1.1)."""
    assert int.from_bytes(frame_bytes[:4], "little") == 0xFD2FB528
    fhd = frame_bytes[4]
    single, did, fcs = (fhd >> 5) & 1, fhd & 3, fhd >> 6
    p = 5 + (0 if single else 1) + [0, 1, 2, 4][did] + [1 if single else 0, 2, 4, 8][fcs]
    bh = int.from_bytes(frame_bytes[p:p + 3], "little")
    if (bh >> 1) & 3 != 2:                             # not a compressed block
        return 0
    lh = frame_bytes[p + 3]
    if lh & 3 != 2:                                    # raw / RLE / treeless literals
        return 0
    return 1 if (lh >> 2) & 3 == 0 else 4


def well_formed_cases():
    """name -> builder of every well-formed case."""
    cases = {
        "rle2_short_repeat": short_repeat_case,
        "rle2_patched_base": patched_base_case,
        "rle2_delta": delta_case,
        "rle2_delta_length_1": delta_one_case,
        "rle1": rle_v1_case,
        "byte_rle": tinyint_case,
        "boolean": boolean_case,
        "decimal_scales_v1": lambda: decimal_case(False),
        "decimal_scales_v2": lambda: decimal_case(True),
        "dictionary_v1": lambda: dictionary_case(False),
        "dictionary_v2": lambda: dictionary_case(True),
        "validity_join": validity_join_case,
        "many_streams": many_streams_case,
    }
    for t in ("BIGINT", "INT", "SMALLINT", "DATE"):
        cases[f"rle2_direct_{t}"] = lambda t=t: direct_case(t)
    for t in ("SMALLINT", "INT", "DATE"):
        cases[f"narrow_{t}"] = lambda t=t: narrow_ints_case(t)
    for t in ("FLOAT", "DOUBLE"):
        cases[f"float_{t}"] = lambda t=t: float_case(t)
    for t in ("STRING", "BINARY"):
        for v2 in (False, True):
            cases[f"direct_{t}_{'v2' if v2 else 'v1'}"] = lambda t=t, v2=v2: direct_strings_case(t, v2)
    for codec, nm in ((ZLIB, "zlib"), (ZSTD, "zstd"), (LZ4, "lz4")):
        cases[f"chunks_{nm}"] = lambda codec=codec: compression_case(codec)[0]
        cases[f"chunks_{nm}_strings"] = lambda codec=codec: compression_case(codec)[1]
    return cases


# ------------------------------------------------------------------ malformed streams
#
# Each returns (OrcFile, vtype).  A decoder that does not check these reads past a stream, writes past its dictionary
# offsets, or (the DECIMAL scale and the dictionary size) loops for as long as a corrupt value says.

def _one(vtype, streams, n, encoding=DIRECT_V2, dict_size=0, codec=NONE, block=262144, values=None, **kw):
    vals = values if values is not None else [0] * n
    return kv_orc_file(VTYPES[vtype], [Stripe(vals, streams, encoding, dict_size)], codec=codec, block=block, **kw), vtype


def _truncated_data():
    """DIRECT run of 100 values at 16 bits (200 bytes) that has lost its last 10 bytes."""
    d, _ = direct(list(range(100)), 15)
    return _one("BIGINT", [Stream(DATA, d[:-10])], 100)


def _truncated_length():
    """DIRECT_V2 strings: 100 rows, the LENGTH stream covers 50."""
    ln, _ = concat(*[short_repeat(2, 1, 10, signed=False) for _ in range(5)])
    return _one("STRING", [Stream(DATA, b"ab" * 100), Stream(LENGTH, ln)], 100)


def _truncated_present():
    """A PRESENT stream that covers 40 of 100 rows."""
    d, _ = direct(list(range(100)), 15)
    return _one("BIGINT", [Stream(PRESENT, bool_stream([True] * 40)), Stream(DATA, d)], 100)


def _dict_id_out_of_range():
    """A dictionary of 4 entries, ids reaching 4."""
    ids, _ = direct([i % 5 for i in range(50)], 2, signed=False)
    ln, _ = short_repeat(1, 1, 4, signed=False)
    return _one("STRING", [Stream(DATA, ids), Stream(LENGTH, ln), Stream(DICTIONARY_DATA, b"abcd")], 50,
                DICTIONARY_V2, 4)


def _dict_lengths_overrun():
    """Dictionary lengths adding up to 20 bytes over a DICTIONARY_DATA stream of 10."""
    ids, _ = short_repeat(0, 1, 10, signed=False)
    ln, _ = short_repeat(5, 1, 4, signed=False)
    return _one("STRING", [Stream(DATA, ids), Stream(LENGTH, ln), Stream(DICTIONARY_DATA, b"0123456789")], 10,
                DICTIONARY_V2, 4)


def _dict_lengths_run_dry():
    """A footer dictionarySize of 8 (within the rows) with a LENGTH stream of 4 entries."""
    ids, _ = short_repeat(0, 1, 10, signed=False)
    ln, _ = short_repeat(1, 1, 4, signed=False)
    return _one("STRING", [Stream(DATA, ids), Stream(LENGTH, ln), Stream(DICTIONARY_DATA, b"abcdefgh")], 10,
                DICTIONARY_V2, 8)


def _dict_size_over_rows(size):
    """A footer that claims a dictionary of `size` entries for a stripe of 10 rows."""
    def make():
        ids, _ = short_repeat(0, 1, 10, signed=False)
        ln, _ = short_repeat(1, 1, 4, signed=False)
        return _one("STRING", [Stream(DATA, ids), Stream(LENGTH, ln), Stream(DICTIONARY_DATA, b"abcd")], 10,
                    DICTIONARY_V2, 4, footer_dict_size={0: size})
    return make


def _patch_index_beyond_run():
    """PATCHED_BASE of 10 values whose patch list lands at index 10."""
    d = patched_base_raw(10, 4, 1, 0, list(range(10)), 8, 8, [10 << 8 | 1])
    return _one("BIGINT", [Stream(DATA, d)], 10)


def _patch_widths_over_64():
    """PATCHED_BASE with a 64-bit patch width and a 2-bit gap width."""
    d = patched_base_raw(10, 4, 1, 0, list(range(10)), 64, 2, [1])
    return _one("BIGINT", [Stream(DATA, d)], 10)


def _chunk_past_stream():
    """A compressed stream whose second chunk header claims more bytes than the stream holds."""
    d, _ = direct(list(range(100)), 15)
    stored = frame(d, ZLIB, 4096) + chunk_header(500, True) + b"x" * 20
    return _one("BIGINT", [Stream(DATA, stored, "asis")], 100, codec=ZLIB, block=4096)


def _chunk_not_inflating(codec):
    """A chunk marked compressed whose bytes are not a valid DEFLATE / zstd / LZ4 block."""
    def make():
        bad = chunk_header(200, False) + bytes([0xFF] * 200)
        return _one("BIGINT", [Stream(DATA, bad, "asis")], 100, codec=codec, block=4096)
    return make


def _decimal_scale(scale, value=1):
    """A DECIMAL(10,5) stripe of 20 rows whose value 7 carries the given per-value scale."""
    def make():
        scales = [5] * 20
        scales[7] = scale
        sec, _ = direct(scales, 31)
        vals = [1] * 20
        vals[7] = value
        return _one("DECIMAL(10,5)", [Stream(DATA, decimal_data(vals)), Stream(SECONDARY, sec)], 20)
    return make


def malformed_cases():
    """name -> builder of (OrcFile, vtype) for each malformed stream or footer the decoder must refuse."""
    return {
        "data_truncated": _truncated_data,
        "length_truncated": _truncated_length,
        "present_truncated": _truncated_present,
        "dict_id_out_of_range": _dict_id_out_of_range,
        "dict_lengths_overrun": _dict_lengths_overrun,
        "dict_lengths_run_dry": _dict_lengths_run_dry,
        "dict_size_over_rows": _dict_size_over_rows(11),
        "dict_size_2e31": _dict_size_over_rows(1 << 31),
        "dict_size_uint32_max": _dict_size_over_rows((1 << 32) - 1),
        "patch_index_beyond_run": _patch_index_beyond_run,
        "patch_widths_over_64": _patch_widths_over_64,
        "chunk_past_stream": _chunk_past_stream,
        "chunk_not_inflating_zlib": _chunk_not_inflating(ZLIB),
        "chunk_not_inflating_zstd": _chunk_not_inflating(ZSTD),
        "chunk_not_inflating_lz4": _chunk_not_inflating(LZ4),
        "decimal_scale_negative_huge": _decimal_scale(-(1 << 62)),
        "decimal_scale_negative": _decimal_scale(-1),
        "decimal_scale_39": _decimal_scale(39),
        "decimal_scale_19_away": _decimal_scale(24),
        "decimal_upscale_overflows": _decimal_scale(0, 10 ** 17),
    }


# ------------------------------------------------------------------ comparison in the expected values' terms

def arrow_values(arr, vt: VType) -> list:
    """pyarrow's reading of "v" as expected values: floats as bit patterns, strings as bytes, decimals unscaled."""
    arr = arr.combine_chunks() if hasattr(arr, "combine_chunks") else arr
    if vt.kind == K_DECIMAL:
        return [None if v is None else int(v.scaleb(vt.scale)) for v in arr.to_pylist()]
    if pa.types.is_date32(arr.type):
        arr = arr.cast(pa.int32())
    if pa.types.is_string(arr.type):                   # (the bytes as stored, UTF-8 or not)
        arr = arr.view(pa.binary())
    valid = arr.is_valid().to_numpy(zero_copy_only=False)
    if vt.kind in (K_FLOAT, K_DOUBLE):
        ub = np.uint32 if vt.width == 4 else np.uint64
        vals = np.asarray(arr.fill_null(0).to_numpy(zero_copy_only=False)).view(ub).tolist()
    else:
        vals = [v.encode() if isinstance(v, str) else v for v in arr.to_pylist()]
    return [v if ok else None for v, ok in zip(vals, valid)]


def read_with_pyarrow(case: Case) -> list:
    import pyarrow.orc as porc
    out = []
    for f in case.files:
        out += arrow_values(porc.ORCFile(io.BytesIO(f.data)).read().column("v"), VTYPES[case.vtype])
    return out


def host_values(col, vt: VType, n: int) -> list:
    """A column of orc_util.decode as expected values."""
    if vt.width == 0:
        data, offs, valid = col
        raw = data.tobytes()
        vals = [raw[offs[i]:offs[i + 1]] for i in range(n)]
    else:
        vals, valid = col
        if vt.kind in (K_FLOAT, K_DOUBLE):
            vals = vals.view(np.uint32 if vt.width == 4 else np.uint64).tolist()
        elif vt.kind == K_BOOLEAN:
            vals = [bool(x) for x in vals.tolist()]
        else:
            vals = vals.tolist()
    return [v if ok else None for v, ok in zip(vals, valid.tolist())]


def first_mismatch(got: list, want: list) -> str:
    if len(got) != len(want):
        return f"{len(got)} values, expected {len(want)}"
    for i, (a, b) in enumerate(zip(got, want)):
        if a != b:
            return f"row {i}: {a!r} != {b!r}"
    return "equal"
