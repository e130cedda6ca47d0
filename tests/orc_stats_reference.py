"""A numpy model of the column statistics the ORC encoder writes (per stripe and per file), and a small protobuf wire
reader that takes them out of an uncompressed ORC file's tail — independent of the library's orc_meta.cc.

The rules restate what OrcSimpleStatsExtractor.toFieldStats (paimon-format/.../orc/filter/
OrcSimpleStatsExtractor.java:119-241) needs from the footer:
  * numberOfValues = the non-null count, hasNull = nulls > 0; a column without non-null values carries nothing else;
    the root column has numberOfValues = rows;
  * integers: {min, max, sum}, the sum exact and left out when it leaves int64; DATE: {min, max};
  * FLOAT / DOUBLE: {min, max} without a sum, a zero min written as -0.0 and a zero max as +0.0, and a stripe or file
    holding a NaN gets [-Infinity, NaN];
  * BOOLEAN: the true count; DECIMAL: {min, max, sum} as decimal strings; STRING / VARCHAR / BINARY: the byte total.
"""
import math
import struct

import numpy as np

INT_KINDS = (1, 2, 3, 4)          # BYTE, SHORT, INT, LONG
FLOAT_KINDS = (5, 6)
BOOLEAN, STRING, BINARY, DECIMAL, DATE, VARCHAR = 0, 7, 8, 14, 15, 16


def decimal_string(unscaled: int, scale: int) -> str:
    neg = unscaled < 0
    digits = str(abs(unscaled))
    if scale > 0:
        digits = digits.rjust(scale + 1, "0")
        digits = digits[:-scale] + "." + digits[-scale:]
    return ("-" if neg else "") + digits


def column_stats(kind, values, valid, scale=0):
    """The expected statistics of one column over some rows.  `values`: a numpy array (fixed width) or a list of bytes
    (var-len); `valid`: bool array."""
    valid = np.asarray(valid, bool)
    n = int(valid.sum())
    out = {"values": n, "has_null": bool((~valid).any())}
    if n == 0:
        return out
    if kind in (STRING, VARCHAR, BINARY):
        out["bytes"] = sum(len(v) for v, ok in zip(values, valid) if ok)
        return out
    v = np.asarray(values)[valid]
    if kind == BOOLEAN:
        out["trues"] = int((v != 0).sum())
    elif kind in FLOAT_KINDS:
        d = v.astype(np.float64)
        if np.isnan(d).any():
            out["min"], out["max"] = -math.inf, math.nan
        else:
            mn, mx = float(d.min()), float(d.max())
            out["min"] = -0.0 if mn == 0 else mn
            out["max"] = 0.0 if mx == 0 else mx
    else:
        ints = [int(x) for x in v]
        out["min"], out["max"] = min(ints), max(ints)
        if kind in INT_KINDS:
            s = sum(ints)
            if -2 ** 63 <= s < 2 ** 63:
                out["sum"] = s
        elif kind == DECIMAL:
            out["min"], out["max"] = decimal_string(out["min"], scale), decimal_string(out["max"], scale)
            out["sum"] = decimal_string(sum(ints), scale)
    return out


def expected(columns, n_rows, stripe_rows):
    """columns: [(kind, values, valid, scale)].  -> (per stripe [root, col...], file [root, col...])"""
    stripe_rows = (stripe_rows + 7) & ~7
    stripes = []
    for g0 in range(0, n_rows, stripe_rows):
        g1 = min(n_rows, g0 + stripe_rows)
        row = [{"values": g1 - g0, "has_null": False}]
        for kind, values, valid, scale in columns:
            row.append(column_stats(kind, values[g0:g1], np.asarray(valid)[g0:g1], scale))
        stripes.append(row)
    whole = [{"values": n_rows, "has_null": False}]
    for kind, values, valid, scale in columns:
        whole.append(column_stats(kind, values, valid, scale))
    return stripes, whole


# ---- protobuf wire reader


def _varint(b, p):
    v = sh = 0
    while True:
        x = b[p]
        p += 1
        v |= (x & 0x7F) << sh
        sh += 7
        if not x & 0x80:
            return v, p


def fields(b):
    """[(field, wire, value)] of one message; length-delimited values are bytes"""
    out, p = [], 0
    while p < len(b):
        key, p = _varint(b, p)
        f, w = key >> 3, key & 7
        if w == 0:
            v, p = _varint(b, p)
        elif w == 1:
            v, p = b[p:p + 8], p + 8
        elif w == 2:
            n, p = _varint(b, p)
            v, p = b[p:p + n], p + n
        elif w == 5:
            v, p = b[p:p + 4], p + 4
        else:
            raise ValueError(f"wire type {w}")
        out.append((f, w, v))
    return out


def _zz(v):
    return (v >> 1) ^ -(v & 1)


def parse_column_statistics(b):
    out = {}
    for f, w, v in fields(b):
        if f == 1:
            out["values"] = v
        elif f == 10:
            out["has_null"] = bool(v)
        elif f in (2, 7):                                    # intStatistics, dateStatistics
            for g, _, x in fields(v):
                out[{1: "min", 2: "max", 3: "sum"}[g]] = _zz(x)
        elif f == 3:                                         # doubleStatistics
            for g, _, x in fields(v):
                out[{1: "min", 2: "max", 3: "sum"}[g]] = struct.unpack("<d", x)[0]
        elif f in (4, 8):                                    # stringStatistics (sum = field 3), binaryStatistics (1)
            for g, _, x in fields(v):
                if (f, g) in ((4, 3), (8, 1)):
                    out["bytes"] = _zz(x)
                else:
                    out[f"string_{g}"] = x
        elif f == 5:                                         # bucketStatistics: packed counts
            for g, gw, x in fields(v):
                out["trues"] = _varint(x, 0)[0] if gw == 2 else x
        elif f == 6:                                         # decimalStatistics
            for g, _, x in fields(v):
                out[{1: "min", 2: "max", 3: "sum"}[g]] = x.decode()
        else:
            out[f"field_{f}"] = v
    return out


def read_tail(blob: bytes):
    """(postscript fields, footer fields, [stripe stats], file stats) of an uncompressed ORC file"""
    ps_len = blob[-1]
    ps = {f: v for f, _, v in fields(blob[-1 - ps_len:-1])}
    assert ps.get(2, 0) == 0, "read_tail reads uncompressed tails"
    footer_len, meta_len = ps[1], ps.get(5, 0)
    foot_end = len(blob) - 1 - ps_len
    footer = fields(blob[foot_end - footer_len:foot_end])
    meta = fields(blob[foot_end - footer_len - meta_len:foot_end - footer_len])
    stripes = [[parse_column_statistics(c) for f, _, c in fields(ss) if f == 1] for f, _, ss in meta if f == 1]
    whole = [parse_column_statistics(v) for f, _, v in footer if f == 7]
    return ps, footer, stripes, whole


def same(got, want):
    """stats equality with NaN == NaN and the sign of zero significant"""
    if set(got) != set(want):
        return False
    for k, w in want.items():
        g = got[k]
        if isinstance(w, float):
            if math.isnan(w):
                if not (isinstance(g, float) and math.isnan(g)):
                    return False
            elif g != w or math.copysign(1, g) != math.copysign(1, w):
                return False
        elif g != w:
            return False
    return True
