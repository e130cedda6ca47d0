"""ORC file tails taken apart and put back together, for tests of the tail reader: the PostScript, Footer and stripe
footers of an uncompressed file as protobuf field lists that a case edits (a length cut or grown, an offset moved past
the end), and the malformed files the decoder must refuse with a format error.

Written from the public ORC specification (file tail: Footer, PostScript, 1-byte PostScript length; orc_proto field
numbers) and the protobuf wire format, independent of the reader in orc_meta.cc."""
import io

import numpy as np
import pyarrow as pa
import pyarrow.orc as orc

from orc_stripes import uvarint

# orc_proto field numbers: PostScript.footerLength, Footer.stripes, StripeInformation.offset / footerLength
PS_FOOTER_LENGTH, FOOTER_STRIPES, SI_OFFSET, SI_FOOTER_LENGTH = 1, 3, 1, 4


def _varint(b: bytes, p: int):
    v, sh = 0, 0
    while True:
        x = b[p]
        p += 1
        v |= (x & 0x7F) << sh
        if not x & 0x80:
            return v, p
        sh += 7


def pb_fields(b: bytes) -> list:
    """A message as [field, wire, value]: an int for wire 0, the raw bytes otherwise."""
    out, p = [], 0
    while p < len(b):
        key, p = _varint(b, p)
        f, w = key >> 3, key & 7
        if w == 0:
            v, p = _varint(b, p)
        elif w == 2:
            n, p = _varint(b, p)
            v, p = b[p:p + n], p + n
        elif w in (1, 5):
            n = 8 if w == 1 else 4
            v, p = b[p:p + n], p + n
        else:
            raise ValueError(f"wire type {w}")
        out.append([f, w, v])
    return out


def pb_bytes(fields: list) -> bytes:
    out = bytearray()
    for f, w, v in fields:
        out += uvarint(f << 3 | w)
        if w == 0:
            out += uvarint(v)
        elif w == 2:
            out += uvarint(len(v)) + bytes(v)
        else:
            out += bytes(v)
    return bytes(out)


class Tail:
    """An uncompressed ORC file as body (magic and stripes) + Footer fields + PostScript fields."""

    def __init__(self, data: bytes):
        ps_len = data[-1]
        self.ps = pb_fields(data[-1 - ps_len:-1])
        flen = self.get(self.ps, PS_FOOTER_LENGTH)
        self.footer = pb_fields(data[-1 - ps_len - flen:-1 - ps_len])
        self.body = data[:-1 - ps_len - flen]

    @staticmethod
    def get(fields, f):
        return next(v for ff, _, v in fields if ff == f)

    @staticmethod
    def set(fields, f, v):
        for x in fields:
            if x[0] == f:
                x[2] = v
                return
        raise KeyError(f)

    def stripes(self) -> list:
        return [pb_fields(v) for f, _, v in self.footer if f == FOOTER_STRIPES]

    def set_stripe(self, i: int, field: int, value: int):
        idx = [k for k, x in enumerate(self.footer) if x[0] == FOOTER_STRIPES][i]
        si = pb_fields(self.footer[idx][2])
        self.set(si, field, value)
        self.footer[idx][2] = pb_bytes(si)

    def build(self, footer: bytes = None, footer_length: int = None, ps: bytes = None) -> bytes:
        """The file again; footer / ps replace the serialized sections, footer_length the PostScript's claim."""
        fb = pb_bytes(self.footer) if footer is None else footer
        if ps is None:
            self.set(self.ps, PS_FOOTER_LENGTH, len(fb) if footer_length is None else footer_length)
            ps = pb_bytes(self.ps)
        assert len(ps) < 256
        return self.body + fb + ps + bytes([len(ps)])


def pyarrow_file(n: int = 3000, seed: int = 0, **opts) -> bytes:
    """A flat file of a few types written by pyarrow.orc."""
    rng = np.random.default_rng(seed)
    t = pa.table({"k": pa.array(np.arange(n, dtype=np.int64)),
                  "v": pa.array(rng.integers(-1000, 1000, n)),
                  "s": pa.array([None if i % 7 == 0 else f"s{i % 97}" for i in range(n)]),
                  "d": pa.array(rng.standard_normal(n))})
    buf = io.BytesIO()
    orc.write_table(t, buf, **opts)
    return buf.getvalue()


def malformed_tails() -> dict:
    """name -> the bytes of a file whose tail is malformed: cut inside its PostScript, its Footer or a stripe footer,
    a Footer length beyond the file (and one that wraps a 64-bit sum), a stripe footer past the end."""
    good = pyarrow_file(4000, stripe_size=4096, compression="uncompressed")
    t = Tail(good)
    assert len(t.stripes()) >= 2
    ps = pb_bytes(t.ps)
    assert ps[0] == PS_FOOTER_LENGTH << 3 and ps[1] & 0x80     # the Footer length varint spans two bytes or more
    footer = pb_bytes(t.footer)
    cases = {
        "postscript_cut_in_footer_length": t.build(ps=ps[:2]),
        "postscript_length_beyond_file": b"ORC" + bytes(40) + bytes([200]),
        "footer_cut": t.build(footer=footer[:len(footer) // 2]),
        "footer_length_beyond_file": t.build(footer_length=len(good) + 100),
        "footer_length_wraps": t.build(footer_length=(1 << 64) - 2),
        "no_magic": b"OXC" + good[3:],
        "three_bytes": b"ORC",
    }
    si = Tail(good)
    si.set_stripe(1, SI_FOOTER_LENGTH, Tail.get(si.stripes()[1], SI_FOOTER_LENGTH) - 1)
    cases["stripe_footer_cut"] = si.build()
    past = Tail(good)
    past.set_stripe(1, SI_FOOTER_LENGTH, len(good))
    cases["stripe_footer_past_end"] = past.build()
    moved = Tail(good)
    moved.set_stripe(0, SI_OFFSET, (1 << 64) - 8)
    cases["stripe_offset_wraps"] = moved.build()
    return cases
