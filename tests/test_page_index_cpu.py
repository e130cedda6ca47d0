"""The page-index model (tests/page_index_reference.py) against its own rules: every truncated STRING / BINARY bound
is a true lower or upper bound, the boundary order, null pages and the NaN rule, the Thrift reader on hand-written
bytes, and the ctypes mirror of pg_parquet_write_options against include/paimon_gpu.h."""
import ctypes as C
import os
import random
import re

import numpy as np
import pytest

import page_index_reference as P
from paimon_b200 import _native as N
from paimon_b200.columnar import Column, KeyValueBatch
from paimon_b200.types import DataField, KeyValueSchema, PhysicalType, RowType

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------- truncation

def _check_bounds(v: bytes, utf8: bool):
    lo, hi = P.truncate_min(v, utf8), P.truncate_max(v, utf8)
    assert lo <= v <= hi, (v, lo, hi)
    if len(v) <= P.TRUNCATE:
        assert lo == v == hi
    else:
        assert len(lo) <= P.TRUNCATE and v.startswith(lo)
        assert hi == v or len(hi) <= P.TRUNCATE + 1
    if utf8:
        lo.decode("utf-8")
        hi.decode("utf-8")
    return lo, hi


def test_random_binary_bounds():
    rng = random.Random(1)
    for _ in range(3000):
        n = rng.choice([0, 1, 63, 64, 65, 66, 100, 300, rng.randrange(0, 200)])
        v = bytes(rng.choice([0, 1, 0x7F, 0x80, 0xFE, 0xFF, rng.randrange(256)]) for _ in range(n))
        _check_bounds(v, False)


@pytest.mark.parametrize("width", [2, 3, 4])
def test_utf8_code_points_straddling_the_cut(width):
    ch = {2: "\u00e9", 3: "\u20ac", 4: "\U0001f600"}[width]
    for lead in range(P.TRUNCATE - 4, P.TRUNCATE + 1):
        for tail in ("", "a", ch * 3):
            v = ("a" * lead + ch + tail).encode()
            lo, hi = _check_bounds(v, True)
            if len(v) > P.TRUNCATE:
                assert len(lo) <= P.TRUNCATE and lo.decode().endswith(("a", ch)) or lo == b""
    rng = random.Random(width)
    alphabet = "aZ~\x7f\u0080\u00e9\u07ff\u0800\u20ac\ud7ff\ue000\uffff\U00010000\U0001f600\U0010fffe\U0010ffff"
    for _ in range(2000):
        s = "".join(rng.choice(alphabet) for _ in range(rng.randrange(0, 80)))
        _check_bounds(s.encode(), True)


def test_max_increments_the_last_position_that_can_be():
    assert P.truncate_max(b"\x01" * 63 + b"\x05" + b"\x00", False) == b"\x01" * 63 + b"\x06"
    assert P.truncate_max(b"\x01" * 62 + b"\x07\xff\x00", False) == b"\x01" * 62 + b"\x08"
    v = b"\xff" * 70
    assert P.truncate_max(v, False) == v                      # nothing can be incremented: the whole value
    assert P.truncate_min(v, False) == b"\xff" * 64
    s = "a" * 63 + "\U0010ffff" + "b"
    assert P.truncate_max(s.encode(), True) == b"a" * 62 + b"b"   # the cut leaves 'a' * 63; its last 'a' becomes 'b'
    s = "\U0010ffff" * 17                                     # 68 bytes, no code point below U+10FFFF
    assert P.truncate_max(s.encode(), True) == s.encode()
    s = "a" * 61 + "\ud7ff" + "x"                             # the increment skips the surrogates
    assert P.truncate_max(s.encode(), True) == ("a" * 61 + "\ue000").encode()
    s = "a" * 63 + "\x7f" + "x"                               # 1 byte -> 2 bytes
    assert P.truncate_max(s.encode(), True) == ("a" * 63 + "\u0080").encode()


# ---------------------------------------------------------------------------------------------- order

def _b(t, vals):
    import stats_reference as S
    return [S.footer_bytes(t, v) for v in vals]


def test_boundary_order():
    T = PhysicalType.INT32
    asc = P.boundary_order(T, [False] * 3, _b(T, [1, 1, 5]), _b(T, [2, 9, 9]))
    desc = P.boundary_order(T, [False] * 3, _b(T, [5, 1, -7]), _b(T, [9, 9, 2]))
    mixed = P.boundary_order(T, [False] * 3, _b(T, [1, 5, 3]), _b(T, [2, 9, 9]))
    crossed = P.boundary_order(T, [False] * 2, _b(T, [1, 0]), _b(T, [2, 3]))   # mins fall, maxes rise
    assert (asc, desc, mixed, crossed) == (P.ASCENDING, P.DESCENDING, P.UNORDERED, P.UNORDERED)
    # signed, not byte order
    assert P.boundary_order(T, [False] * 2, _b(T, [-1, 1]), _b(T, [-1, 1])) == P.ASCENDING
    # null pages do not take part; one or no non-null page is ASCENDING; equal pages are ASCENDING
    assert P.boundary_order(T, [False, True, False], _b(T, [1, 0, 2]), _b(T, [1, 0, 2])) == P.ASCENDING
    assert P.boundary_order(T, [True, True], [b"", b""], [b"", b""]) == P.ASCENDING
    assert P.boundary_order(T, [False], _b(T, [3]), _b(T, [3])) == P.ASCENDING
    assert P.boundary_order(T, [False] * 2, _b(T, [3, 3]), _b(T, [4, 4])) == P.ASCENDING
    # floats numerically (-0.0 == +0.0), bytes unsigned with a proper prefix first
    D = PhysicalType.DOUBLE
    assert P.boundary_order(D, [False] * 2, _b(D, [-0.0, 0.0]), _b(D, [0.0, 0.0])) == P.ASCENDING
    assert P.boundary_order(D, [False] * 2, _b(D, [-2.5, -3.0]), _b(D, [1e300, -1.0])) == P.DESCENDING
    S_ = PhysicalType.STRING
    assert P.boundary_order(S_, [False] * 3, [b"a", b"ab", b"\xc3"], [b"a", b"b", b"\xff"]) == P.ASCENDING
    assert P.boundary_order(S_, [False] * 2, [b"\x80", b"\x7f"], [b"\x80", b"\x7f"]) == P.DESCENDING


def _schema(*fields):
    vt = RowType(tuple(DataField(n, t, nullable) for n, t, nullable in fields))
    return KeyValueSchema.of(vt, [fields[0][0]])


def _batch(schema, cols):
    n = len(cols[0])
    from test_stats_reference_cpu import column
    keys = column(PhysicalType.INT64, list(range(n)))
    seq = Column(PhysicalType.INT64, np.arange(n, dtype=np.int64))
    kinds = Column(PhysicalType.INT8, np.zeros(n, np.int8))
    out = [keys, seq, kinds]
    for f, vals in zip(schema.value_type.fields, cols):
        valid = np.array([v is not None for v in vals])
        fill = [0 if v is None else v for v in vals] if f.physical not in (PhysicalType.STRING, PhysicalType.BINARY) \
            else vals
        out.append(column(f.physical, fill, valid))
    return KeyValueBatch(schema, out)


def test_null_pages_nan_rule_and_zero_rule():
    schema = _schema(("k", "BIGINT", False), ("d", "DOUBLE", True), ("f", "FLOAT", True), ("s", "STRING", True))
    d = [None] * 8 + [0.0, -0.0, 1.5, None, 0.0, 0.0, 0.0, 0.0] + [2.0, float("nan")] + [1.0] * 6
    f = [None] * 8 + [-0.0] * 8 + [0.0] * 8
    s = [None] * 8 + ["b", "a", None, "c"] + ["x"] * 4 + ["\u00e9" * 40] * 8
    b = _batch(schema, [list(range(24)), d, f, s])
    idx = P.page_index(b, page_rows=8, row_group_rows=16)
    assert len(idx) == 2 and [len(ci.pages) for ci in idx[0]] == [2] * 7
    D, F, S_ = 4, 5, 6
    ci = idx[0][D].column_index
    assert ci.null_pages == [True, False] and ci.null_counts == [8, 1]
    assert ci.min_values[0] == b"" and ci.min_values[1] == np.float64(-0.0).tobytes()
    assert ci.max_values[1] == np.float64(1.5).tobytes()
    assert idx[1][D].column_index is None and idx[1][D].pages == [(0, 8)]      # a NaN: no ColumnIndex
    ci = idx[0][F].column_index
    assert ci.min_values[1] == np.float32(-0.0).tobytes() and ci.max_values[1] == np.float32(0.0).tobytes()
    ci = idx[0][S_].column_index
    assert ci.min_values == [b"", b"a"] and ci.max_values == [b"", b"x"] and ci.null_counts == [8, 1]
    long = ("\u00e9" * 40).encode()                                # 80 bytes, a 2-byte character across byte 64
    ci = idx[1][S_].column_index
    assert ci.min_values == [long[:64]] and ci.max_values == [("\u00e9" * 31 + "\u00ea").encode()]
    assert idx[0][0].column_index.boundary_order == P.ASCENDING
    assert [p for p, _ in idx[1][0].pages] == [0]


def test_slices_start_their_row_groups_at_row0():
    schema = _schema(("k", "BIGINT", False), ("i", "INT", True))
    b = _batch(schema, [list(range(40)), [None if r % 5 == 0 else 40 - r for r in range(40)]])
    idx = P.page_index(b, row0=8, n_rows=30, page_rows=8, row_group_rows=16)
    assert [ci.pages for ci in (idx[0][4], idx[1][4])] == [[(0, 8), (8, 8)], [(0, 8), (8, 6)]]
    ci = idx[0][4].column_index                               # rows 8..23, NULL at 10, 15 and 20
    assert ci.boundary_order == P.DESCENDING and ci.null_counts == [2, 1]
    assert ci.min_values[0] == (40 - 14).to_bytes(4, "little") and ci.max_values[0] == (40 - 8).to_bytes(4, "little")


# ---------------------------------------------------------------------------------------------- Thrift reader

def test_thrift_reader_on_hand_written_bytes():
    # ColumnIndex {1: [true, false], 2: ["", "a"], 3: ["", "b"], 4: 1, 5: [3, 0]}
    b = bytes([0x19, 0x21, 1, 2, 0x19, 0x28, 0, 1, ord("a"), 0x19, 0x28, 0, 1, ord("b"), 0x15, 2, 0x19, 0x26, 6, 0, 0])
    assert P.parse_column_index(b) == P.ColumnIndex([True, False], [b"", b"a"], [b"", b"b"], 1, [3, 0])
    # OffsetIndex {1: [{1: 4, 2: 100, 3: 0}, {1: 104, 2: 20, 3: 64}]}
    b = bytes([0x19, 0x2C, 0x16, 8, 0x15, 200, 1, 0x16, 0, 0, 0x16, 208, 1, 0x15, 40, 0x16, 128, 1, 0, 0])
    assert P.parse_offset_index(b) == [(4, 100, 0), (104, 20, 64)]
    with pytest.raises(AssertionError):
        P.parse_offset_index(b + b"\x00")


# ---------------------------------------------------------------------------------------------- ABI

def test_write_options_mirror_the_header():
    src = open(os.path.join(ROOT, "include", "paimon_gpu.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} pg_parquet_write_options;", src).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"(int64_t|int32_t)\s+(\w+);", body)
    assert fields == [("int64_t", "row_group_rows"), ("int64_t", "page_rows"), ("int64_t", "page_index")]
    assert [f[0] for f in N.PgParquetWriteOptions._fields_] == [f[1] for f in fields]
    assert C.sizeof(N.PgParquetWriteOptions) == 24
    assert [getattr(N.PgParquetWriteOptions, f[1]).offset for f in fields] == [0, 8, 16]
    assert N.PgParquetWriteOptions(0, 0).page_index == 0                  # the default: no page index
